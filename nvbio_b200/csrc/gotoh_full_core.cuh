// gotoh_full_core.cuh -- full-matrix (un-banded) Gotoh scoring, one alignment per thread (SURVEY 8f-3).
//
// Semantics: aln::alignment_score with GotohAligner<TYPE,scheme,PatternBlockingTag>
// (nvbio/alignment/gotoh/gotoh_inl.h:459-960): rows follow the TEXT, columns the PATTERN; E runs along the pattern and
// F along the text, both with the PATTERN gap costs; first column H = text_gap_open + i*text_gap_ext for GLOBAL else 0,
// E = 0 for LOCAL else -inf (:75-89); top row H = Go + (j-1)*Ge for GLOBAL and SEMI_GLOBAL, 0 for LOCAL, F = -inf
// (:688-696); -inf = SHRT_MIN - min(Go,Ge) (:665).  sink = (text end, pattern end).  LOCAL reports every cell in stripes
// of 8 pattern columns (gotoh_bandlen_selector, :1491-1495), row by row inside a stripe, so a tie resolves to the last
// maximal cell in (stripe, row, column) order; SEMI_GLOBAL reports H[i][M] of every row, GLOBAL H[N][M].
//
// Formulation here: 32-column pattern stripes held in registers, the text swept once per stripe, the stripe's right-hand
// boundary column (H,E per text row) kept in HBM scratch between stripes; four 8-column LOCAL trackers per stripe merged
// in order reproduce the reference's tie-breaking exactly.
#pragma once
#include "gotoh_core.cuh"

namespace nvb {

constexpr int FULL_W = 32;     // pattern columns per stripe

// DIRS: also emit the 4-bit direction vector of every cell (H source | E extended | F extended; the bits
// GotohSubmatrixContext::new_cell stores, gotoh_inl.h:426-446) to dirs[row * dir_row_words + stripe * 4 ..]: one uint4 per
// (text row, 32-column stripe), nibble k of word w = pattern column 32*stripe + 8*w + k.
template <int TYPE, bool DIRS, bool QUAL>
__host__ __device__ inline SinkResult gotoh_full_impl2(const GotohScheme& S,
        const uint32_t* __restrict__ pwords, uint32_t pbits, uint32_t pbe, uint32_t poff, uint32_t M,
        const uint32_t* __restrict__ twords, uint32_t tbits, uint32_t tbe, uint32_t toff, uint32_t N,
        int2* __restrict__ col, size_t col_stride, uint32_t* __restrict__ dirs = nullptr, uint32_t dir_row_words = 0,
        const uint8_t* __restrict__ quals = nullptr)
{
    SinkResult res; res.score = NVB_SINK_MIN; res.x = 0xFFFFFFFFu; res.y = 0xFFFFFFFFu;
    if (M == 0 || N == 0) return res;            // outside the supported domain (see header)
    const int32_t Go = S.pgo, Ge = S.pge;
    const int32_t INF = SHRT_MIN - (Go < Ge ? Go : Ge);

    for (uint32_t b = 0; b < M; b += FULL_W) {
        const bool first = (b == 0), last = (b + FULL_W >= M);
        uint32_t q[FULL_W];
        uint32_t qq4[FULL_W / 4];                 // the stripe's base qualities, four per word (quality-table schemes only)
        {
            SymReaderRT pr(pwords, pbits, pbe);
#pragma unroll
            for (int j = 0; j < FULL_W; ++j) q[j] = (b + j < M) ? pr.get(poff + b + j) : 256u;     // 256 never equals a text symbol
#pragma unroll
            for (int w = 0; w < FULL_W / 4; ++w) qq4[w] = 0u;
            if (QUAL && quals) {
#pragma unroll
                for (int j = 0; j < FULL_W; ++j) if (b + j < M) qq4[j >> 2] |= (uint32_t)quals[poff + b + j] << (8 * (j & 3));
            }
        }
        int32_t H[FULL_W + 1], F[FULL_W + 1];
#pragma unroll
        for (int j = 0; j <= FULL_W; ++j) {
            H[j] = (TYPE != NVB_LOCAL) ? ((b + j > 0) ? Go + Ge * (int32_t)(b + j - 1) : 0) : 0;
            F[j] = INF;
        }
        int32_t diag_next = H[0];                                    // H[0][b]
        int32_t tb[4] = { INT_MIN, INT_MIN, INT_MIN, INT_MIN };      // LOCAL trackers of the four 8-column sub-stripes
        uint32_t tp[4] = { 0, 0, 0, 0 };                             // (row << 16) | column, 1-based
        SymReaderRT tr(twords, tbits, tbe);
        for (uint32_t r = 0; r < N; ++r) {
            const uint32_t g = tr.get(toff + r);
            int32_t Hl, E;
            if (first) { Hl = (TYPE == NVB_GLOBAL) ? S.tgo + S.tge * (int32_t)r : 0; E = (TYPE == NVB_LOCAL) ? 0 : INF; }
            else       { const int2 c = col[(size_t)r * col_stride]; Hl = c.x; E = c.y; }
            int32_t Hd = diag_next;
            diag_next = Hl;
            H[0] = Hl;
            uint32_t dw[4] = { 0u, 0u, 0u, 0u };
#pragma unroll
            for (int j = 1; j <= FULL_W; ++j) {
                const int32_t ftop = F[j] + Ge, htop = H[j] + Go;         // H[j] still holds the previous row
                F[j] = imax2(ftop, htop);
                const int32_t eleft = E + Ge, hleft = H[j - 1] + Go;      // H[j-1] is already this row
                E    = imax2(eleft, hleft);
                int32_t sub = (g == q[j - 1]) ? S.match : S.mismatch;
                if (QUAL) sub = S.qtab[2u * ((qq4[(j - 1) >> 2] >> (8 * ((j - 1) & 3))) & 255u) + ((g == q[j - 1]) ? 0u : 1u)];
                const int32_t diagonal = Hd + sub;
                int32_t h = imax2(imax2(E, F[j]), diagonal);
                if (TYPE == NVB_LOCAL) h = imax2(h, 0);
                if (DIRS) {
                    const int32_t top = F[j], left = E;
                    uint32_t d = top > left ? (top > diagonal ? (uint32_t)DIR_DEL : (uint32_t)DIR_SUB) : (left > diagonal ? (uint32_t)DIR_INS : (uint32_t)DIR_SUB);
                    if (TYPE == NVB_LOCAL && h == 0) d = DIR_SINK;
                    d |= (eleft > hleft ? (uint32_t)DIR_INS_EXT : 0u) | (ftop > htop ? (uint32_t)DIR_DEL_EXT : 0u);
                    dw[(j - 1) >> 3] |= d << (4 * ((j - 1) & 7));
                }
                Hd = H[j];
                H[j] = h;
                if (TYPE == NVB_LOCAL && b + (uint32_t)j <= M) {
                    const int k = (j - 1) >> 3;
                    if (tb[k] <= h) { tb[k] = h; tp[k] = ((r + 1u) << 16) | (b + (uint32_t)j); }
                }
            }
            if (!last) col[(size_t)r * col_stride] = make_int2(H[FULL_W], E);
            if (DIRS) {
                uint32_t* dp = dirs + (size_t)r * dir_row_words + (b / FULL_W) * 4u;
                dp[0] = dw[0]; dp[1] = dw[1]; dp[2] = dw[2]; dp[3] = dw[3];
            }
            if (TYPE == NVB_SEMI_GLOBAL && last) {
                int32_t hM = H[1];
#pragma unroll
                for (int j = 1; j <= FULL_W; ++j) if (b + (uint32_t)j == M) hM = H[j];
                if (res.score <= hM) { res.score = hM; res.x = r + 1u; res.y = M; }
            }
        }
        if (TYPE == NVB_GLOBAL && last) {
            int32_t hM = H[1];
#pragma unroll
            for (int j = 1; j <= FULL_W; ++j) if (b + (uint32_t)j == M) hM = H[j];
            res.score = hM; res.x = N; res.y = M;
        }
        if (TYPE == NVB_LOCAL) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (b + 8u * (uint32_t)k < M && res.score <= tb[k]) { res.score = tb[k]; res.x = tp[k] >> 16; res.y = tp[k] & 0xFFFFu; }
        }
    }
    return res;
}

// quality tables (a table look-up per cell) are compiled as a separate instantiation so that constant schemes do not pay for them
template <int TYPE, bool DIRS>
__host__ __device__ inline SinkResult gotoh_full_impl(const GotohScheme& S,
        const uint32_t* __restrict__ pwords, uint32_t pbits, uint32_t pbe, uint32_t poff, uint32_t M,
        const uint32_t* __restrict__ twords, uint32_t tbits, uint32_t tbe, uint32_t toff, uint32_t N,
        int2* __restrict__ col, size_t col_stride, uint32_t* __restrict__ dirs = nullptr, uint32_t dir_row_words = 0,
        const uint8_t* __restrict__ quals = nullptr)
{
    if (S.qtab) return gotoh_full_impl2<TYPE, DIRS, true>(S, pwords, pbits, pbe, poff, M, twords, tbits, tbe, toff, N, col, col_stride, dirs, dir_row_words, quals);
    return gotoh_full_impl2<TYPE, DIRS, false>(S, pwords, pbits, pbe, poff, M, twords, tbits, tbe, toff, N, col, col_stride, dirs, dir_row_words, quals);
}

template <int TYPE>
__host__ __device__ inline SinkResult gotoh_full(const GotohScheme& S,
        const uint32_t* __restrict__ pwords, uint32_t pbits, uint32_t pbe, uint32_t poff, uint32_t M,
        const uint32_t* __restrict__ twords, uint32_t tbits, uint32_t tbe, uint32_t toff, uint32_t N,
        int2* __restrict__ col, size_t col_stride, const uint8_t* __restrict__ quals = nullptr)
{
    return gotoh_full_impl<TYPE, false>(S, pwords, pbits, pbe, poff, M, twords, tbits, tbe, toff, N, col, col_stride, nullptr, 0, quals);
}

// direction nibble of cell (text row r, pattern column c), both 0-based, in gotoh_full_impl2's row-major layout
struct FullDirsRowMajor {
    const uint32_t* __restrict__ dirs; uint32_t row_words;
    __host__ __device__ __forceinline__ uint32_t operator()(uint32_t r, uint32_t c) const {
        return (dirs[(size_t)r * row_words + (c >> 3)] >> (4u * (c & 7u))) & 15u;
    }
};

// walk the direction matrix from the sink (state machine of nvbio/alignment/gotoh/gotoh_inl.h:1806-1871 plus the first-row /
// first-column completion of the generic driver, alignment_inl.h:452-471); ops in END -> START order, returns their number.
// `dir(r, c)` is the direction nibble of cell (text row r, pattern column c), both 0-based (FullDirsRowMajor, FullDirsStepMajor)
template <int TYPE, class Dirs>
__host__ __device__ inline uint32_t gotoh_full_walk(const Dirs& dir, const SinkResult& sink,
                                                    uint8_t* __restrict__ ops, uint32_t max_ops, uint32_t& src_x, uint32_t& src_y)
{
    int32_t row = (int32_t)sink.x, col = (int32_t)sink.y - 1;          // row 1-based over the text, col 0-based over the pattern
    uint32_t n_ops = 0, state = 0;                                      // HSTATE 0, ESTATE 1, FSTATE 2
    while (row > 0 && col >= 0) {
        const uint32_t op = dir((uint32_t)(row - 1), (uint32_t)col);
        const uint32_t h_op = op & 3u;
        if (TYPE == NVB_LOCAL && state == 0 && h_op == DIR_SINK) break;
        if (state == 1)      { if ((op & DIR_INS_EXT) == 0) state = 0; --col; if (n_ops < max_ops) ops[n_ops] = DIR_INS; ++n_ops; }
        else if (state == 2) { if ((op & DIR_DEL_EXT) == 0) state = 0; --row; if (n_ops < max_ops) ops[n_ops] = DIR_DEL; ++n_ops; }
        else {
            if (h_op == DIR_INS) state = 1;
            else if (h_op == DIR_DEL) state = 2;
            else { --row; --col; if (n_ops < max_ops) ops[n_ops] = DIR_SUB; ++n_ops; }
        }
    }
    uint32_t sx = (uint32_t)row, sy = (uint32_t)(col + 1);
    if (TYPE != NVB_LOCAL && sx == 0u) for (; sy > 0u; --sy) { if (n_ops < max_ops) ops[n_ops] = DIR_INS; ++n_ops; }
    if (TYPE == NVB_GLOBAL && sy == 0u) for (; sx > 0u; --sx) { if (n_ops < max_ops) ops[n_ops] = DIR_DEL; ++n_ops; }
    src_x = sx; src_y = sy;
    return n_ops;
}
// the same over gotoh_full_impl2's row-major matrix of `dir_row_words` words per text row
template <int TYPE>
__host__ __device__ inline uint32_t gotoh_full_walk(const uint32_t* __restrict__ dirs, uint32_t dir_row_words, const SinkResult& sink,
                                                    uint8_t* __restrict__ ops, uint32_t max_ops, uint32_t& src_x, uint32_t& src_y)
{
    return gotoh_full_walk<TYPE>(FullDirsRowMajor{dirs, dir_row_words}, sink, ops, max_ops, src_x, src_y);
}

// ---------------------------------------------------------------------------------------------
// warp-per-alignment full-matrix traceback (gotoh_full_warp_traceback_kernel, gotoh_kernels.cu).  Lane l owns pattern columns
// [l*W, l*W + W) and computes text row t - l at step t, the left boundary (H, E) of its row arriving from lane l - 1 (a wavefront, as in
// gotoh_full_warp_kernel).  int32, with the recurrence and direction bits of gotoh_full_impl2<TYPE, true, QUAL>.  The W nibbles of one
// lane and step are NW = ceil(W / 8) words, stored step-major: word w of lane l at step t is dirs[(t * NW + w) * 32 + l] (one coalesced
// 128-byte row per step and word).
// ---------------------------------------------------------------------------------------------
struct FullDirsStepMajor {
    const uint32_t* __restrict__ dirs; uint32_t w, nw;                  // columns per lane, words per lane and step
    __host__ __device__ __forceinline__ uint32_t operator()(uint32_t r, uint32_t c) const {
        const uint32_t l = c / w, k = c - l * w;                        // lane, column within the lane; the lane computed row r at step r + l
        return (dirs[((size_t)(r + l) * nw + (k >> 3)) * 32u + l] >> (4u * (k & 7u))) & 15u;
    }
};

template <int W>
struct FullTbLane {
    static constexpr int NW = (W + 7) / 8;
    uint32_t q[W];                 // the lane's pattern symbols (256 past the pattern's end: never equal to a text symbol)
    int32_t s_eq[W], s_ne[W];      // their substitution scores on a match / mismatch (the quality table's, when the scheme has one)
    int32_t H[W], F[W];            // H and F of the previous row in the lane's columns
    int32_t Hd;                    // H of the previous row in the column left of the lane's first one

    // top row of the lane's columns c0 + 1 .. c0 + W (1-based) of a pattern of M symbols at offset poff
    template <int TYPE>
    __host__ __device__ __forceinline__ void init(const GotohScheme& S, const uint32_t* __restrict__ pwords, uint32_t pbits, uint32_t pbe,
                                                  uint32_t poff, uint32_t M, const uint8_t* __restrict__ quals, uint32_t c0, int32_t INF)
    {
#pragma unroll
        for (int k = 0; k < W; ++k) {
            const uint32_t c = c0 + (uint32_t)k;
            q[k] = c < M ? sym_at_rt(pwords, pbits, pbe, poff + c) : 256u;
            const uint32_t qq = (S.qtab && quals && c < M) ? (uint32_t)quals[poff + c] : 0u;
            s_eq[k] = S.qtab ? S.qtab[2u * qq] : S.match;
            s_ne[k] = S.qtab ? S.qtab[2u * qq + 1u] : S.mismatch;
            H[k] = (TYPE != NVB_LOCAL) ? S.pgo + S.pge * (int32_t)c : 0;
            F[k] = INF;
        }
        Hd = (TYPE != NVB_LOCAL && c0 > 0u) ? S.pgo + S.pge * (int32_t)(c0 - 1u) : 0;
    }

    // one row against text symbol g: (Hl, E) = the row's H and E left of the lane's first column on entry, in its last column on exit
    template <int TYPE>
    __host__ __device__ __forceinline__ void row(const GotohScheme& S, uint32_t g, int32_t& Hl, int32_t& E, uint32_t (&dw)[NW])
    {
        const int32_t Go = S.pgo, Ge = S.pge;
        int32_t hd = Hd;
        Hd = Hl;
#pragma unroll
        for (int w = 0; w < NW; ++w) dw[w] = 0u;
#pragma unroll
        for (int k = 0; k < W; ++k) {
            const int32_t ftop = F[k] + Ge, htop = H[k] + Go;
            F[k] = imax2(ftop, htop);
            const int32_t eleft = E + Ge, hleft = Hl + Go;
            E = imax2(eleft, hleft);
            const int32_t diagonal = hd + ((g == q[k]) ? s_eq[k] : s_ne[k]);
            int32_t h = imax2(imax2(E, F[k]), diagonal);
            if (TYPE == NVB_LOCAL) h = imax2(h, 0);
            const int32_t top = F[k], left = E;
            uint32_t d = top > left ? (top > diagonal ? (uint32_t)DIR_DEL : (uint32_t)DIR_SUB) : (left > diagonal ? (uint32_t)DIR_INS : (uint32_t)DIR_SUB);
            if (TYPE == NVB_LOCAL && h == 0) d = DIR_SINK;
            d |= (eleft > hleft ? (uint32_t)DIR_INS_EXT : 0u) | (ftop > htop ? (uint32_t)DIR_DEL_EXT : 0u);
            dw[k >> 3] |= d << (4 * (k & 7));
            hd = H[k];
            H[k] = h;
            Hl = h;
        }
    }
};

// The warp traceback's outputs: item i = (alignment a, output slot `out`) writes ops[out * max_ops ..], n_ops[out] and source[out] =
// (text begin, pattern begin); the text begin is relative to a's text, or with `absolute` its offset in the text set's words
struct FullTbOut { uint8_t* ops; uint32_t* n_ops; uint2* source; uint32_t max_ops; uint32_t absolute; };
struct FullTbArgs {
    GotohScheme S; StrSet pat, txt; const uint8_t* quals;
    const int32_t* score; const uint2* sink;           // every alignment's score and sink (the score pass's)
    const uint2* items; const uint32_t* n_items;       // the alignments to trace, their count on the device
    FullTbOut o; void* pool;
};
constexpr uint32_t FULL_TB_MAX_M = 512u;               // 16 pattern columns per lane
// gotoh_kernels.cu: with a == NULL only *pool_bytes (the slot pool, bounded by the resident warps and max_n, not by the item count);
// else the launch.  NVB_E_UNSUPPORTED unless 1 <= max_m <= FULL_TB_MAX_M and max_n <= 65535
int full_warp_traceback(int type, uint32_t max_m, uint32_t max_n, const FullTbArgs* a, size_t* pool_bytes, cudaStream_t s);
// gotoh_kernels.cu: nvb_banded_gotoh_traceback over the first min(*d_n, n) alignments, the count on the device (d_n == NULL: all n); the
// temp size is that of n alignments
int banded_traceback(int band_len, int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals,
                     const nvb_string_set* texts, const uint32_t* d_n, uint32_t n, int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                     uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops, void* d_temp, size_t* temp_bytes, void* stream);

// left boundary (H, E) of text row r (0-based) in the first column, as gotoh_full_impl2 starts its first stripe
template <int TYPE>
__host__ __device__ __forceinline__ void full_first_column(const GotohScheme& S, uint32_t r, int32_t INF, int32_t& Hl, int32_t& E)
{
    Hl = (TYPE == NVB_GLOBAL) ? S.tgo + S.tge * (int32_t)r : 0;
    E = (TYPE == NVB_LOCAL) ? 0 : INF;
}

// ---------------------------------------------------------------------------------------------
// packed pair: TWO full-matrix alignments per thread in s16x2 halves (DPX), same formulation as gotoh_pair (gotoh_core.cuh)
// transposed: the per-ROW substitution profile comes from the two text symbols, the per-COLUMN selector from the two
// pattern symbols (constant over a stripe sweep; staged by the thread itself in `sel`, element j at sel[j*sel_stride] --
// shared memory on the device: one conflict-free u16 column per thread, read back with one LDS.U16 per cell).
//
// Preconditions (the caller routes everything else to gotoh_full): M0 == M1 >= 1, N0 == N1 >= 1, every pattern symbol < 4
// (returns false otherwise, before touching any output), scheme admitted by full_pair_path_ok().
// LOCAL keeps H itself (>= 0, < 2048) and F,E biased by beta = -Go; per row the maximum of the 16-bit keys
// (H << 5) | (column within the stripe) is taken, and since the column index is (8-column sub-stripe << 3) | column, comparing
// keys >> 3 across rows and whole keys inside a row reproduces the reference's (sub-stripe, row, column) report order.
// ---------------------------------------------------------------------------------------------
static inline bool full_pair_path_ok(int type, const nvb_gotoh_scheme* s, uint32_t max_m, uint32_t max_n) {
    const int64_t Go = s->pattern_gap_open, Ge = s->pattern_gap_ext;
    if (Go >= 0 || Ge >= 0 || s->text_gap_open >= 0 || s->text_gap_ext >= 0) return false;
    int64_t s_lo = s->match < s->mismatch ? s->match : s->mismatch, s_hi = s->match > s->mismatch ? s->match : s->mismatch;
    if (s->d_qual_table) {                               // quality-dependent scores: the caller's bounds on the table's values
        if (s->qual_table_min == 0 && s->qual_table_max == 0) return false;      // unknown: the int32 kernel
        s_lo = s->qual_table_min; s_hi = s->qual_table_max;
    }
    int64_t mx = s_lo < 0 ? -s_lo : s_lo; if (s_hi > mx) mx = s_hi; if (-s_hi > mx) mx = -s_hi;
    if (-Go > mx) mx = -Go; if (-Ge > mx) mx = -Ge;
    if (-(int64_t)s->text_gap_open > mx) mx = -(int64_t)s->text_gap_open;
    if (-(int64_t)s->text_gap_ext > mx) mx = -(int64_t)s->text_gap_ext;
    if (((int64_t)max_m + (int64_t)max_n + 4) * mx > 30000) return false;          // every intermediate fits 16 bits
    if (s_lo - Go < -128 || s_hi - Go > 127) return false;                          // (S - Go) is looked up as an int8
    if (type == NVB_LOCAL) {
        const uint32_t mn = max_m < max_n ? max_m : max_n;
        if ((int64_t)mn * (s_hi > 0 ? s_hi : 0) >= 2048) return false;              // key = (H << 5) | column in 16 bits
    }
    return true;
}

// sequential symbol reader over a packed string (one shift per symbol, one load per word)
struct SymSeq {
    const uint32_t* wp; uint32_t w, left, bits, be, spw;
    __host__ __device__ __forceinline__ SymSeq(const uint32_t* words, uint32_t b, uint32_t e, uint32_t off)
        : bits(b), be(b == 8 ? 0u : e), spw(32u / b) {
        const uint32_t lg = (b == 2 ? 4u : (b == 4 ? 3u : 2u));
        const uint32_t r = off & (spw - 1u);
        wp = words + (off >> lg);
        w = *wp++;
        if (r) w = be ? (w << (bits * r)) : (w >> (bits * r));
        left = spw - r;
    }
    __host__ __device__ __forceinline__ uint32_t next() {
        if (left == 0u) { w = *wp++; left = spw; }
        const uint32_t s = be ? (w >> (32u - bits)) : (w & ((1u << bits) - 1u));
        w = be ? (w << bits) : (w >> bits);
        --left;
        return s;
    }
};

struct FullPairTrack { int32_t k0, k1; uint32_t r0, r1; int32_t s0, s1; uint32_t x0, x1; };   // LOCAL: best key/row; SEMI: best score/row

// per-row state of the packed full-matrix stripe: left neighbour / diagonal / E of the cell being computed, the row's sink bookkeeping
struct FullRow { uint32_t Vl, Vd, E, rowkey, vM, vlast; };
struct FullConsts { uint32_t Ge2, Go2, GoX, beta2, keymul; };

// one cell (column j = 1..FULL_W of the stripe) of text row R; V[j] / F[j] hold the previous row's values on entry and this row's on exit
// QUAL (quality-dependent substitution scores, nvBowtie's scheme): the score depends on the pattern COLUMN's base quality, so the
// roles are swapped -- `colp` holds two 4-byte profiles per column (indexed by the TEXT symbol) and P0 carries the row's selector
template <int TYPE, bool PARTIAL, bool QUAL>
__host__ __device__ __forceinline__ void full_pair_cell(const int j, uint32_t (&V)[FULL_W + 1], uint32_t (&F)[FULL_W + 1], FullRow& R,
        const uint32_t P0, const uint32_t P1, const uint16_t* sel, const uint32_t* colp, const uint32_t sel_stride, const uint32_t ncols, const FullConsts& K)
{
    const uint32_t s = QUAL ? prmt(colp[(size_t)(2 * (j - 1)) * sel_stride], colp[(size_t)(2 * (j - 1) + 1) * sel_stride], P0)
                            : prmt(P0, P1, (uint32_t)sel[(size_t)(j - 1) * sel_stride]);
    F[j] = NVB_VIADDMAX(F[j], K.Ge2, V[j]);
    R.E  = NVB_VIADDMAX(R.E, K.Ge2, (j == 1) ? R.Vl : V[j - 1]);
    const uint32_t old = V[j];
    if (TYPE == NVB_LOCAL) {
        const uint32_t hb = NVB_VIMAX3(NVB_VIADDMAX(R.Vd, s, F[j]), R.E, K.beta2);
        V[j] = hb + K.GoX;                                                    // H = h' + Go per half, one 32-bit add (carry-free)
        const uint32_t key = V[j] * K.keymul + (uint32_t)((j - 1) | ((j - 1) << 16));   // IMAD
        if (!PARTIAL || (uint32_t)j <= ncols) R.rowkey = NVB_VIMAX_U(R.rowkey, key);
    } else {
        const uint32_t h = NVB_VIMAX(NVB_VIADDMAX(R.Vd, s, F[j]), R.E);
        V[j] = NVB_VIADD(h, K.Go2);
        if (TYPE == NVB_SEMI_GLOBAL && PARTIAL && (uint32_t)j == ncols) R.vM = V[j];
    }
    if (j == FULL_W) R.vlast = V[j];
    R.Vd = old;
}

// Two text rows per loop iteration, the second one two columns behind the first (the same idea as in the banded kernel, gotoh_core.cuh:
// a row is one serial chain E -> h' -> H; two rows in flight give a thread two independent chains).  The in-place V[] / F[] update
// stays valid: row r+1 reads column j only after row r has written it, and keeps its own diagonal (the value it overwrote).
template <int TYPE, bool PARTIAL, bool QUAL>
__host__ __device__ __forceinline__ void full_pair_stripe(const GotohScheme& S, const bool first, const bool last, const uint32_t b,
        const uint32_t ncols, const uint32_t N, SymSeq t0, SymSeq t1, const uint16_t* sel, const uint32_t* colp, const uint32_t sel_stride,
        uint2* __restrict__ col, const size_t col_stride, FullPairTrack& trk, uint32_t& g_last, const uint32_t* prof_tab, uint32_t& bad_text)
{
    const int32_t Go = S.pgo, Ge = S.pge;
    int32_t INF = SHRT_MIN - (Go < Ge ? Go : Ge);
    if (INF + Ge < -32768) INF = -32768 - Ge;
    const int32_t c_eq = S.match - Go, c_ne = S.mismatch - Go;
    const int32_t beta = -Go;
    FullConsts K;
    K.Ge2 = pack16(Ge, Ge); K.Go2 = pack16(Go, Go); K.GoX = (uint32_t)(Go * 65537); K.beta2 = pack16(beta, beta); K.keymul = S.keymul;
    const uint32_t INFx = (TYPE == NVB_LOCAL) ? pack16(INF + beta, INF + beta) : pack16(INF, INF);

    // arrays of the PREVIOUS row: V[j] = H (LOCAL) or H + Go (otherwise) of column b + j; F[j] likewise biased for LOCAL
    uint32_t V[FULL_W + 1], F[FULL_W + 1];
#pragma unroll
    for (int j = 0; j <= FULL_W; ++j) {
        int32_t h = 0;
        if (TYPE != NVB_LOCAL) h = ((b + j > 0) ? Go + Ge * (int32_t)(b + j - 1) : 0) + Go;
        V[j] = pack16(h, h);
        F[j] = INFx;
    }
    uint32_t diag_next = V[0];
    uint32_t left_h = (TYPE == NVB_LOCAL) ? 0u : pack16(((TYPE == NVB_GLOBAL) ? S.tgo : 0) + Go, ((TYPE == NVB_GLOBAL) ? S.tgo : 0) + Go);
    const uint32_t left_step = (TYPE == NVB_GLOBAL) ? pack16(S.tge, S.tge) : 0u;
    const uint32_t left_e = (TYPE == NVB_LOCAL) ? K.beta2 : INFx;

    // the boundary column (H, E) of the stripe to the left, fetched one row pair ahead of its use
    uint2 nA = make_uint2(0u, 0u), nB = nA;
    if (!first) { nA = col[0]; if (N > 1u) nB = col[col_stride]; }
#define NVB_FULL_ROW_BEGIN(R, c_)                                                                               \
    {   if (first) { R.Vl = left_h; R.E = left_e; left_h = NVB_VIADD(left_h, left_step); }                      \
        else       { R.Vl = c_.x; R.E = c_.y; }                                                                 \
        R.Vd = diag_next; diag_next = R.Vl; R.rowkey = 0u; R.vM = 0u; R.vlast = 0u; }
#define NVB_FULL_ROW_END(R, r)                                                                                  \
    {   if (!last) col[(size_t)(r) * col_stride] = make_uint2(R.vlast, R.E);                                    \
        if (TYPE == NVB_LOCAL) {                                                                                \
            const int32_t k0 = (int32_t)(R.rowkey & 0xFFFFu), k1 = (int32_t)(R.rowkey >> 16);                   \
            if (k0 >= (trk.k0 & ~7)) { trk.k0 = k0; trk.r0 = (r); }   /* (H, sub-stripe) >= the best's: later rows win ties */ \
            if (k1 >= (trk.k1 & ~7)) { trk.k1 = k1; trk.r1 = (r); }                                             \
        }                                                                                                       \
        if (TYPE == NVB_SEMI_GLOBAL && last) {                                                                  \
            const uint32_t vm_ = PARTIAL ? R.vM : R.vlast;                                                      \
            const int32_t h0 = half_lo(vm_) - Go, h1 = half_hi(vm_) - Go;                                       \
            if (trk.s0 <= h0) { trk.s0 = h0; trk.x0 = (r) + 1u; }                                               \
            if (trk.s1 <= h1) { trk.s1 = h1; trk.x1 = (r) + 1u; }                                               \
        } }

    constexpr int SK = 2;
    uint32_t r = 0;
    for (; r + 1u < N; r += 2u) {
        const uint32_t ga0 = t0.next(), ga1 = t1.next(), gb0 = t0.next(), gb1 = t1.next();
        uint32_t PA0, PA1, PB0, PB1;
        if (QUAL) {                                   // row selectors from the text symbols (a text symbol > 3 has no selector: the caller bails out)
            bad_text |= (ga0 | ga1 | gb0 | gb1) >> 2;
            PA0 = pair_selector(ga0 & 3u, ga1 & 3u); PB0 = pair_selector(gb0 & 3u, gb1 & 3u); PA1 = PB1 = 0u;
        } else {
            PA0 = prof_tab ? prof_tab[ga0] : sub_profile(ga0, c_eq, c_ne); PA1 = prof_tab ? prof_tab[ga1] : sub_profile(ga1, c_eq, c_ne);
            PB0 = prof_tab ? prof_tab[gb0] : sub_profile(gb0, c_eq, c_ne); PB1 = prof_tab ? prof_tab[gb1] : sub_profile(gb1, c_eq, c_ne);
        }
        FullRow A, B;
        NVB_FULL_ROW_BEGIN(A, nA)
        NVB_FULL_ROW_BEGIN(B, nB)
        if (!first) {
            if (r + 2u < N) nA = col[(size_t)(r + 2u) * col_stride];
            if (r + 3u < N) nB = col[(size_t)(r + 3u) * col_stride];
        }
#pragma unroll
        for (int jj = 1; jj <= FULL_W + SK; ++jj) {
            if (jj <= FULL_W) full_pair_cell<TYPE, PARTIAL, QUAL>(jj,      V, F, A, PA0, PA1, sel, colp, sel_stride, ncols, K);
            if (jj > SK)      full_pair_cell<TYPE, PARTIAL, QUAL>(jj - SK, V, F, B, PB0, PB1, sel, colp, sel_stride, ncols, K);
        }
        V[0] = B.Vl;
        NVB_FULL_ROW_END(A, r)
        NVB_FULL_ROW_END(B, r + 1u)
    }
    if (r < N) {
        const uint32_t g0 = t0.next(), g1 = t1.next();
        uint32_t P0, P1;
        if (QUAL) { bad_text |= (g0 | g1) >> 2; P0 = pair_selector(g0 & 3u, g1 & 3u); P1 = 0u; }
        else      { P0 = prof_tab ? prof_tab[g0] : sub_profile(g0, c_eq, c_ne); P1 = prof_tab ? prof_tab[g1] : sub_profile(g1, c_eq, c_ne); }
        FullRow A;
        NVB_FULL_ROW_BEGIN(A, nA)
#pragma unroll
        for (int j = 1; j <= FULL_W; ++j) full_pair_cell<TYPE, PARTIAL, QUAL>(j, V, F, A, P0, P1, sel, colp, sel_stride, ncols, K);
        V[0] = A.Vl;
        NVB_FULL_ROW_END(A, r)
    }
#undef NVB_FULL_ROW_BEGIN
#undef NVB_FULL_ROW_END
    if (TYPE == NVB_GLOBAL && last) {
        uint32_t v = V[FULL_W];
        if (PARTIAL) {
#pragma unroll
            for (int j = 1; j <= FULL_W; ++j) if ((uint32_t)j == ncols) v = V[j];
        }
        g_last = v;
    }
}

// QUAL: `colp` (two words per stripe column, same stride as `sel`) replaces `sel`; `quals` = one base quality per pattern symbol at
// the symbols' own offsets (NULL: quality 0 everywhere); S.qtab is the 256 x 2 table.  A pattern N is then simply a column whose
// profile is all-mismatch; a text symbol > 3 makes the routine return false (the caller scores the pair with the int32 kernel).
template <int TYPE, bool QUAL = false>
__host__ __device__ inline bool gotoh_full_pair(const GotohScheme& S,
        const uint32_t* __restrict__ pwords, uint32_t pbits, uint32_t pbe, uint32_t poff0, uint32_t poff1, uint32_t M,
        const uint32_t* __restrict__ twords, uint32_t tbits, uint32_t tbe, uint32_t toff0, uint32_t toff1, uint32_t N,
        uint2* __restrict__ col, size_t col_stride, uint16_t* sel, uint32_t sel_stride, SinkResult& r0, SinkResult& r1,
        const uint32_t* prof_tab = nullptr,      // optional 256-entry table of sub_profile(g, c_eq, c_ne) (shared memory on the device)
        uint32_t* colp = nullptr, const uint8_t* __restrict__ quals = nullptr)
{
    const int32_t Go = S.pgo;
    r0.score = NVB_SINK_MIN; r0.x = r0.y = 0xFFFFFFFFu; r1 = r0;
    FullPairTrack trk; trk.s0 = trk.s1 = INT_MIN; trk.x0 = trk.x1 = 0u;
    uint32_t bad_text = 0u;
    for (uint32_t b = 0; b < M; b += FULL_W) {
        const bool first = (b == 0), last = (b + FULL_W >= M);
        const uint32_t ncols = last ? M - b : (uint32_t)FULL_W;
        {
            SymSeq p0(pwords, pbits, pbe, poff0 + b), p1(pwords, pbits, pbe, poff1 + b);
            uint32_t bad = 0u;
#pragma unroll
            for (int j = 0; j < FULL_W; ++j) {
                uint32_t q0 = 0u, q1 = 0u;
                if ((uint32_t)j < ncols) { q0 = p0.next(); q1 = p1.next(); }
                if (QUAL) {
                    const uint32_t qq0 = (quals && (uint32_t)j < ncols) ? quals[poff0 + b + j] : 0u;
                    const uint32_t qq1 = (quals && (uint32_t)j < ncols) ? quals[poff1 + b + j] : 0u;
                    colp[(size_t)(2 * j) * sel_stride]     = sub_profile(q0, S.qtab[2 * qq0] - Go, S.qtab[2 * qq0 + 1] - Go);
                    colp[(size_t)(2 * j + 1) * sel_stride] = sub_profile(q1, S.qtab[2 * qq1] - Go, S.qtab[2 * qq1 + 1] - Go);
                } else {
                    bad |= (q0 | q1) >> 2;
                    sel[(size_t)j * sel_stride] = (uint16_t)pair_selector(q0 & 3u, q1 & 3u);
                }
            }
            if (bad) return false;            // a pattern symbol >= 4 (N): not expressible as a 2-bit selector
        }
        trk.k0 = trk.k1 = -1; trk.r0 = trk.r1 = 0u;
        uint32_t g_last = 0u;
        const SymSeq t0(twords, tbits, tbe, toff0), t1(twords, tbits, tbe, toff1);
        if (ncols == (uint32_t)FULL_W) full_pair_stripe<TYPE, false, QUAL>(S, first, last, b, ncols, N, t0, t1, sel, colp, sel_stride, col, col_stride, trk, g_last, prof_tab, bad_text);
        else                           full_pair_stripe<TYPE, true,  QUAL>(S, first, last, b, ncols, N, t0, t1, sel, colp, sel_stride, col, col_stride, trk, g_last, prof_tab, bad_text);
        if (QUAL && bad_text) return false;                     // an N in the text: no row selector for it
        if (TYPE == NVB_LOCAL) {
            if (r0.score <= (trk.k0 >> 5)) { r0.score = trk.k0 >> 5; r0.x = trk.r0 + 1u; r0.y = b + ((uint32_t)trk.k0 & 31u) + 1u; }
            if (r1.score <= (trk.k1 >> 5)) { r1.score = trk.k1 >> 5; r1.x = trk.r1 + 1u; r1.y = b + ((uint32_t)trk.k1 & 31u) + 1u; }
        }
        if (TYPE == NVB_GLOBAL && last) {
            r0.score = half_lo(g_last) - Go; r0.x = N; r0.y = M;
            r1.score = half_hi(g_last) - Go; r1.x = N; r1.y = M;
        }
    }
    if (TYPE == NVB_SEMI_GLOBAL) {
        r0.score = trk.s0; r0.x = trk.x0; r0.y = M;
        r1.score = trk.s1; r1.x = trk.x1; r1.y = M;
    }
    return true;
}

} // namespace nvb
