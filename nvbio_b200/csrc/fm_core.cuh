// fm_core.cuh -- per-thread FM-index primitives over the interleaved {bwt,occ} 32-byte blocks.
//
// Behaviour follows nvbio (paths relative to the reference tree):
//   rank_dictionary_inl.h:424-538   dispatch_rank<2,64,PackedStream<...,2,true>,...,uint4,uint4>
//   popcount_inl.h:239-247,327-350  popc_2bit / truncated popc_2bit
//   fmindex_inl.h:36-99             `$`-aware rank(fmi,k,c) / rank(fmi,range,c)
//   fmindex_inl.h:307-341           match();   mapping_inl.h:83-97 match_range (N -> (1,0))
//   fmindex_inl.h:471-499           locate();  ssa_inl.h:487-504 SSA_index_multiple_context<16>
// The code is a fresh formulation: one 32-byte sector per block (two adjacent 128-bit loads on sm_90a), a
// branch-free prefix popcount over the four BWT words, and a uniform treatment of the reference's
// special cases (k==-1, k==length, primary shift), which are all pure functions of (k,c).
#pragma once
#include "common.cuh"

namespace nvb {

struct __align__(32) FmBlock {
    uint32_t bwt[4];   // 64 symbols, 2-bit big-endian: symbol s of word q at bits [31-2s, 30-2s]
    uint32_t occ[4];   // #A,#C,#G,#T in bwt[0, 64k)
};

struct FmIndex {
    const FmBlock*  blocks;
    const uint32_t* ssa;
    const uint2*    ktab;          // optional k-mer range table (NULL = none)
    uint32_t n, primary;
    uint32_t L2[5];
    uint32_t sa_mask, sa_shift;    // sampled-SA interval I = 1 << sa_shift, mask = I - 1
    uint32_t ktab_k;
    uint32_t ktab_located;         // 1: table entries are 16 bytes {x, y, SA[x], SA[y]} (SA values filled for ranges of one or two rows; nvb_fm_build_ktab_located)
                                   // 2: the same, and the last word of a ONE-row entry holds the 16 text symbols before SA[x] (nvb_fm_build_ktab_context)
    const uint2*    rows;          // optional, with a context table: {SA[r], the 16 text symbols before SA[r]} for every row r (nvb_fm_build_rows;
                                   // nvb_fm_index.ktab_located == 3 or 5, which is 2 here plus this array)
    uint32_t ktab_wide;            // 1: 32-byte entries (nvb_fm_build_ktab_wide; nvb_fm_index.ktab_located 4 / 5, ktab_located 2 here): the first
                                   // 16 bytes as at level 2, k-mers with 3 to 8 occurrences also carry their rows' contexts (see ktab_wide_fill)
    // constant-index selects keep the struct in the kernel-parameter constant bank (a dynamic L2[c]
    // would force a local-memory copy of the whole struct)
    __host__ __device__ __forceinline__ uint32_t l2(uint32_t c) const {
        return (c == 0) ? L2[0] : (c == 1) ? L2[1] : (c == 2) ? L2[2] : L2[3];
    }
    __host__ __device__ __forceinline__ uint32_t count(uint32_t c) const {
        return (c == 0) ? L2[1] - L2[0] : (c == 1) ? L2[2] - L2[1] : (c == 2) ? L2[3] - L2[2] : L2[4] - L2[3];
    }
};

static inline bool valid_fmindex(const nvb_fm_index* f) {
    if (!f || !f->d_bwt_occ || f->length > NVB_FM_MAX_LENGTH) return false;
    const uint32_t I = f->sa_interval;
    if (I != 0 && (I & (I - 1)) != 0) return false;           // power of two
    if (f->d_ktab && (f->ktab_k < 1 || f->ktab_k > 16 || f->ktab_located > 5u)) return false;
    if (f->d_ktab && f->ktab_located >= 3u && (f->sa_interval != 1u || !f->d_ssa)) return false;
    if (f->d_ktab && f->ktab_located >= 4u && ((uintptr_t)f->d_ktab & 31u)) return false;
    if (f->d_ktab && (f->ktab_located == 3u || f->ktab_located == 5u) && !f->d_rows) return false;
    return true;
}
static inline FmIndex make_fmindex(const nvb_fm_index* f) {
    FmIndex r;
    r.blocks = (const FmBlock*)f->d_bwt_occ; r.ssa = f->d_ssa; r.n = f->length; r.primary = f->primary;
    for (int i = 0; i < 5; ++i) r.L2[i] = f->L2[i];
    const uint32_t I = f->sa_interval ? f->sa_interval : 16u;
    r.sa_shift = 0; while ((1u << r.sa_shift) < I) ++r.sa_shift;
    r.sa_mask = (1u << r.sa_shift) - 1u;
    r.ktab = (const uint2*)f->d_ktab; r.ktab_k = f->d_ktab ? f->ktab_k : 0u;
    // d_rows is read only at levels 3 and 5: callers that fill the struct field by field and stop at ktab_located leave it undefined
    const bool with_rows = f->d_ktab && (f->ktab_located == 3u || f->ktab_located == 5u);
    r.ktab_wide = (f->d_ktab && f->ktab_located >= 4u) ? 1u : 0u;
    r.ktab_located = f->d_ktab ? (f->ktab_located >= 2u ? 2u : f->ktab_located) : 0u;
    r.rows = with_rows ? (const uint2*)f->d_rows : nullptr;
    return r;
}

__host__ __device__ __forceinline__ uint32_t nvb_popc(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// L2 fetch granularity of the block gathers: a plain load pulls the whole 128-byte line from DRAM (4 sectors per gather for
// the 32 useful bytes); ".L2::64B" asks for half of it.
#ifndef NVB_FM_LD_QUAL
#define NVB_FM_LD_QUAL ".L2::64B"
#endif
__host__ __device__ __forceinline__ FmBlock load_block(const FmBlock* __restrict__ blocks, uint32_t k) {
#ifdef __CUDA_ARCH__
    // sm_90a has no 256-bit load: the 32-byte block (one sector, 32-byte aligned) is two 128-bit read-only loads issued back to back
    // in one asm statement (volatile keeps paired loads adjacent)
    FmBlock b;
    asm volatile("ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(b.bwt[0]), "=r"(b.bwt[1]), "=r"(b.bwt[2]), "=r"(b.bwt[3]),
                   "=r"(b.occ[0]), "=r"(b.occ[1]), "=r"(b.occ[2]), "=r"(b.occ[3])
                 : "l"(blocks + k));
    return b;
#else
    return blocks[k];
#endif
}
// b = blocks[k] if pred (else b is left untouched); issued right behind a preceding load_block so that
// both gathers of an LF step are in flight together
__host__ __device__ __forceinline__ void load_block_if(FmBlock& b, const FmBlock* __restrict__ blocks, uint32_t k, bool pred) {
#ifdef __CUDA_ARCH__
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %9, 0;\n\t"
                 "@p ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "@p ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%4,%5,%6,%7}, [%8+16];\n\t}"
                 : "+r"(b.bwt[0]), "+r"(b.bwt[1]), "+r"(b.bwt[2]), "+r"(b.bwt[3]),
                   "+r"(b.occ[0]), "+r"(b.occ[1]), "+r"(b.occ[2]), "+r"(b.occ[3])
                 : "l"(blocks + k), "r"((uint32_t)pred));
#else
    if (pred) b = blocks[k];
#endif
}

// scattered 4- and 8-byte gathers (SA entries, k-mer table entries): like the block gathers they ask L2 for 64 bytes of the line
// instead of all 128 (a plain LDG drags the whole line from DRAM for 8 useful bytes)
__host__ __device__ __forceinline__ uint32_t gather_u32(const uint32_t* __restrict__ p) {
#ifdef __CUDA_ARCH__
    uint32_t v; asm volatile("ld.global.nc" NVB_FM_LD_QUAL ".u32 %0, [%1];" : "=r"(v) : "l"(p)); return v;
#else
    return *p;
#endif
}
__host__ __device__ __forceinline__ uint4 gather_u4(const uint4* __restrict__ p) {
#ifdef __CUDA_ARCH__
    uint4 v; asm volatile("ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v;
#else
    return *p;
#endif
}
__host__ __device__ __forceinline__ uint2 gather_u2(const uint2* __restrict__ p) {
#ifdef __CUDA_ARCH__
    uint2 v; asm volatile("ld.global.nc" NVB_FM_LD_QUAL ".v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p)); return v;
#else
    return *p;
#endif
}

// one-hot flags (at bit 30-2s) of the symbols of w equal to c
__host__ __device__ __forceinline__ uint32_t eq_flags(uint32_t w, uint32_t pat) {
    const uint32_t d = w ^ pat;
    return ~(d | (d >> 1)) & 0x55555555u;
}

// occurrences of c among symbols [0, r] (r in 0..63) of the block, plus the block's base counter:
// = rank(dict, 64k + r, c)
__host__ __device__ __forceinline__ uint32_t block_rank(const FmBlock& b, uint32_t r, uint32_t c) {
    const uint32_t pat = c * 0x55555555u;
    const uint32_t nsym = r + 1;                              // 1..64 symbols to keep
    uint32_t cnt = (c == 0) ? b.occ[0] : (c == 1) ? b.occ[1] : (c == 2) ? b.occ[2] : b.occ[3];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        // symbols of word q to keep: clamp(nsym - 16q, 0, 16), counted from the top of the word
        const int keep = (int)nsym - 16 * q;
        const uint32_t k = keep < 0 ? 0u : (keep > 16 ? 16u : (uint32_t)keep);
        const uint32_t mask = (uint32_t)(0xFFFFFFFF00000000ull >> (2 * k));
        cnt += nvb_popc(eq_flags(b.bwt[q], pat) & mask);
    }
    return cnt;
}

__host__ __device__ __forceinline__ uint32_t block_symbol(const FmBlock& b, uint32_t r) {
    const uint32_t q = r >> 4;
    const uint32_t w = (q == 0) ? b.bwt[0] : (q == 1) ? b.bwt[1] : (q == 2) ? b.bwt[2] : b.bwt[3];
    return (w >> (30u - 2u * (r & 15u))) & 3u;
}

// ---------------------------------------------------------------------------------------------
// generic rank dictionary (SURVEY 8a row a6): the reference's dispatch_rank for a PLAIN big-endian 2-bit PackedStream over
// 32- or 64-bit words with a separate occurrence table sampled every K symbols, 32- or 64-bit counters
// (rank_dictionary_inl.h:243-422; the form its tests and 64-bit indices use).  rank(dict, i, c) = #c in text[0, i];
// i == all-ones -> 0.  K is a multiple of the symbols per word.
// ---------------------------------------------------------------------------------------------
template <typename W> struct dict_word {};
template <> struct dict_word<uint32_t> { static constexpr uint32_t SPW = 16u; static constexpr uint32_t ODD = 0x55555555u; };
template <> struct dict_word<uint64_t> { static constexpr uint32_t SPW = 32u; static constexpr uint64_t ODD = 0x5555555555555555ull; };

// occurrences of c among the first `keep` symbols (1..SPW) of word w
template <typename W>
__host__ __device__ __forceinline__ uint32_t word_rank(W w, uint32_t c, uint32_t keep) {
    constexpr uint32_t SPW = dict_word<W>::SPW;
    const W pat = (W)c * dict_word<W>::ODD;
    const W d = w ^ pat;
    W flags = ~(d | (d >> 1)) & dict_word<W>::ODD;
    flags &= (W)(~(W)0) << (2u * (SPW - keep));
#ifdef __CUDA_ARCH__
    return sizeof(W) == 8 ? (uint32_t)__popcll((unsigned long long)flags) : (uint32_t)__popc((uint32_t)flags);
#else
    return (uint32_t)__builtin_popcountll((unsigned long long)flags);
#endif
}
template <typename W, typename I>
__host__ __device__ __forceinline__ I dict_rank(const W* __restrict__ text, const I* __restrict__ occ, uint32_t K, I i, uint32_t c) {
    if (i == (I)(~(I)0)) return (I)0;
    constexpr uint32_t SPW = dict_word<W>::SPW;
    const uint64_t k = (uint64_t)(i / K);
    const uint32_t r = (uint32_t)(i - (I)(k * K));               // offset inside the block, 0..K-1
    const uint32_t m = r / SPW;
    const uint64_t off = k * (K / SPW);
    I out = occ[k * 4u + c];
    for (uint32_t j = 0; j < m; ++j) out += word_rank<W>(text[off + j], c, SPW);
    return out + word_rank<W>(text[off + m], c, (r % SPW) + 1u);
}

// rank(fmi, k, c)  (fmindex_inl.h:36-57)
__host__ __device__ __forceinline__ uint32_t fm_rank1(const FmIndex& f, uint32_t k, uint32_t c) {
    if (k == 0xFFFFFFFFu) return 0u;
    if (k == f.n) return f.count(c);
    if (k >= f.primary) --k;
    const FmBlock b = load_block(f.blocks, k >> 6);
    return block_rank(b, k & 63u, c);
}

// rank4(fmi, k): occurrences of all four symbols in rows [0,k]  (fmindex_inl.h:107-133 ->
// rank_dictionary_inl.h:539-550 run4 with the count table; here four masked popcounts of the same block)
__host__ __device__ __forceinline__ uint4 fm_rank4(const FmIndex& f, uint32_t k) {
    if (k == 0xFFFFFFFFu) return make_uint4(0u, 0u, 0u, 0u);
    if (k == f.n) return make_uint4(f.count(0), f.count(1), f.count(2), f.count(3));
    if (k >= f.primary) --k;
    const FmBlock b = load_block(f.blocks, k >> 6);
    const uint32_t r = k & 63u;
    return make_uint4(block_rank(b, r, 0), block_rank(b, r, 1), block_rank(b, r, 2), block_rank(b, r, 3));
}

// rank(fmi, (kx,ky), c)  (fmindex_inl.h:66-99 -> rank_dictionary_inl.h:512-538).  All of the
// reference's case splits reduce to "each end is rank1 of that end"; the only thing worth keeping
// is the shared block load when both ends fall in one 64-symbol block.
__host__ __device__ __forceinline__ void fm_rank2(const FmIndex& f, uint32_t kx, uint32_t ky, uint32_t c,
                                                  uint32_t& rx, uint32_t& ry) {
    const bool need_x = (kx != 0xFFFFFFFFu) && (kx != f.n);
    const bool need_y = (ky != 0xFFFFFFFFu) && (ky != f.n);
    const uint32_t cnt = f.count(c);
    rx = (kx == f.n) ? cnt : 0u;
    ry = (ky == f.n) ? cnt : 0u;
    const uint32_t ax = kx - (kx >= f.primary ? 1u : 0u);
    const uint32_t ay = ky - (ky >= f.primary ? 1u : 0u);
    if (need_x || need_y) {
        const uint32_t bx = ax >> 6, by = ay >> 6;
        FmBlock b0 = load_block(f.blocks, need_x ? bx : by);
        FmBlock b1 = b0;
        load_block_if(b1, f.blocks, by, need_x && need_y && bx != by);
        const uint32_t tx = block_rank(b0, ax & 63u, c);
        const uint32_t ty = block_rank(b1, ay & 63u, c);
        if (need_x) rx = tx;
        if (need_y) ry = ty;
    }
}

// one backward-search step; returns false when the range became empty
__host__ __device__ __forceinline__ void fm_step(const FmIndex& f, uint32_t c, uint32_t& x, uint32_t& y) {
    uint32_t rx, ry;
    fm_rank2(f, x - 1u, y, c, rx, ry);
    const uint32_t base = f.l2(c);
    x = base + rx + 1u;
    y = base + ry;
}

// symbols [a, a + cnt) (1 <= cnt <= 16) of a 2-bit big-endian stream in the TOP 2*cnt bits of the result (the low bits are
// unspecified); touches the second word only when the window really reaches into it
__host__ __device__ __forceinline__ uint32_t be2_window(const uint32_t* __restrict__ words, uint32_t a, uint32_t cnt)
{
    const uint32_t wi = a >> 4, r = a & 15u;
    const uint32_t w0 = words[wi];
    if (r == 0u) return w0;
    const uint32_t w1 = (r + cnt > 16u) ? words[wi + 1u] : 0u;
    return (w0 << (2u * r)) | (w1 >> (32u - 2u * r));
}

// Context tables (ktab_located == 2) of an index with fewer than 0xC0000000 rows pack a TWO-row entry {x, x + 1, SA[x], SA[x + 1]} as
// {x, 0xC0000000 | ctxA | ctxB << 14, SA[x], SA[x + 1]}: y = x + 1 is implied (no valid row index reaches 0xC0000000) and the freed
// bits hold the 7 text symbols before SA[x] (ctxA) and before SA[x + 1] (ctxB), last symbol in the lowest two bits
constexpr uint32_t KTAB_TWO_ROW_MARK = 0xC0000000u;
__host__ __device__ __forceinline__ bool ktab_two_row_marker(const FmIndex& f, const uint32_t y) {
    return f.ktab_located == 2u && f.n < KTAB_TWO_ROW_MARK && y >= KTAB_TWO_ROW_MARK;
}

// the (up to) `want` text symbols before pos, symbol pos-1 in the lowest two bits (none for the `$` row, pos symbols when pos < want)
__host__ __device__ __forceinline__ uint32_t text_before(const uint32_t* __restrict__ text, const uint32_t pos, const uint32_t want)
{
    const uint32_t cnt = (pos == 0xFFFFFFFFu) ? 0u : (pos < want ? pos : want);
    return cnt ? (be2_window(text, pos - cnt, cnt) >> (32u - 2u * cnt)) : 0u;
}

// Wide context tables (nvb_fm_build_ktab_wide): 32-byte entries w[0..7], one DRAM sector, whose first 16 bytes are the level-2 entry for
// k-mers with at most two occurrences and the empty range.  A k-mer with 3 to KTAB_WIDE_ROWS occurrences (rows x..y) also carries, in
// the words that level 2 leaves zero:
//     3 rows:     {x, y, SA[x], SA[x+1], SA[x+2], ctx16(x), ctx16(x+1), ctx16(x+2)}
//     4 rows:     {x, y, ctx8(x) | ctx8(x+1) << 16, ctx8(x+2) | ctx8(x+3) << 16, SA[x], SA[x+1], SA[x+2], SA[x+3]}
//     5-8 rows:   {x, y, ctx8 of rows x, x+1 | x+2, x+3 | ... (two per word, words 2..5), 0, ...}
// ctxN(r) = the N text symbols before SA[r] (text_before).  Wider ranges are {x, y, 0, ...}.
constexpr uint32_t KTAB_WIDE_ROWS = 8;
__host__ __device__ __forceinline__ void ktab_wide_fill(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ text, uint32_t n,
                                                        uint32_t x, uint32_t y, uint32_t (&w)[8])
{
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = 0u;
    w[0] = x; w[1] = y;
    if (x > y) return;
    const uint32_t d = y - x;
    if (d == 0u) { w[2] = sa[x]; w[3] = text_before(text, w[2], 16u); return; }
    if (d == 1u) {
        w[2] = sa[x]; w[3] = sa[y];
        if (n < KTAB_TWO_ROW_MARK) w[1] = KTAB_TWO_ROW_MARK | text_before(text, w[2], 7u) | (text_before(text, w[3], 7u) << 14);
        return;
    }
    if (d == 2u) {
#pragma unroll
        for (int i = 0; i < 3; ++i) { w[2 + i] = sa[x + i]; w[5 + i] = text_before(text, w[2 + i], 16u); }
        return;
    }
    if (d >= KTAB_WIDE_ROWS) return;
#pragma unroll
    for (uint32_t i = 0; i < KTAB_WIDE_ROWS; ++i) {
        if (i > d) continue;
        const uint32_t pos = sa[x + i];
        w[2 + i / 2u] |= text_before(text, pos, 8u) << (16u * (i & 1u));
        if (d == 3u) w[4 + i] = pos;
    }
}
// row x + i of a wide entry {lo, hi} with 3 (`three`) or 4..8 rows: its context (16 or 8 symbols) and, for 3 or 4 rows, its SA value
__host__ __device__ __forceinline__ uint32_t ktab_wide_context(const uint4& lo, const uint4& hi, bool three, uint32_t i)
{
    if (three) return i == 0u ? hi.y : (i == 1u ? hi.z : hi.w);
    const uint32_t w = i < 2u ? lo.z : (i < 4u ? lo.w : (i < 6u ? hi.x : hi.y));
    return (i & 1u) ? (w >> 16) : (w & 0xFFFFu);
}
__host__ __device__ __forceinline__ uint32_t ktab_wide_sa(const uint4& lo, const uint4& hi, bool three, uint32_t i)
{
    if (three) return i == 0u ? lo.z : (i == 1u ? lo.w : hi.x);
    return i == 0u ? hi.x : (i == 1u ? hi.y : (i == 2u ? hi.z : hi.w));
}

// the k-mer table entry u: 16 bytes into lo, and with a wide table the other 16 bytes of its sector into hi (else hi is left untouched),
// both loads issued together
__host__ __device__ __forceinline__ void gather_ktab_entry(const FmIndex& f, uint32_t u, uint4& lo, uint4& hi)
{
    const uint4* p = (const uint4*)f.ktab + ((uint64_t)u << f.ktab_wide);        // 4^16 x 32 B does not fit 32 bits
#ifdef __CUDA_ARCH__
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %9, 0;\n\t"
                 "ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "@p ld.global.nc" NVB_FM_LD_QUAL ".v4.u32 {%4,%5,%6,%7}, [%8+16];\n\t}"
                 : "=r"(lo.x), "=r"(lo.y), "=r"(lo.z), "=r"(lo.w), "+r"(hi.x), "+r"(hi.y), "+r"(hi.z), "+r"(hi.w)
                 : "l"(p), "r"(f.ktab_wide));
#else
    lo = p[0];
    if (f.ktab_wide) hi = p[1];
#endif
}

// match() of one query read through a SymReader; FORWARD consumes left-to-right, COMPLEMENT maps
// c<4 -> 3-c (nvBowtie's reverse-complement seed search over the forward index).
template <int BITS, bool BE>
__host__ __device__ __forceinline__ void fm_match_one(const FmIndex& f, const uint32_t* __restrict__ words,
                                                      uint32_t off, uint32_t len, uint32_t flags,
                                                      uint32_t& ox, uint32_t& oy) {
    SymReader<BITS, BE> rd(words);
    uint32_t x = 0, y = f.n;
    const bool fwd = (flags & NVB_MATCH_FORWARD_ORDER) != 0;
    const bool comp = (flags & NVB_MATCH_COMPLEMENT) != 0;
    uint32_t s = 0;
    if (f.ktab_k && len >= f.ktab_k) {
        // the first k symbols consumed are the LAST k symbols of the effective pattern: look their range up.
        // ktab[u] is match() of that k-mer, which also reproduces the reference's early exit on an empty range.
        uint32_t u = 0; bool has_n = false;
        if (BITS == 2 && BE && !fwd) {
            // backward order over a 2-bit big-endian stream: the index is the bit pattern of the last k symbols (complemented: ~)
            const uint32_t w = be2_window(words, off + len - f.ktab_k, f.ktab_k);
            u = (comp ? ~w : w) >> (32u - 2u * f.ktab_k);
        } else {
            for (uint32_t j = 0; j < f.ktab_k; ++j) {
                const uint32_t i = fwd ? j : (len - 1u - j);
                uint32_t c = rd.get(off + i);
                has_n |= (c > 3u);
                if (comp) c = 3u - c;
                u |= (c & 3u) << (2u * j);
            }
        }
        if (!has_n) {                                   // an N among them: take the step-by-step path below
            // (ranges only: the first 8 bytes of a 16- or 32-byte entry)
            const uint2 r = gather_u2(f.ktab_located ? (const uint2*)((const uint4*)f.ktab + ((uint64_t)u << f.ktab_wide)) : f.ktab + u);
            x = r.x; y = ktab_two_row_marker(f, r.y) ? r.x + 1u : r.y; s = f.ktab_k;
        }
    }
    for (; s < len && x <= y; ++s) {
        const uint32_t i = fwd ? s : (len - 1u - s);
        uint32_t c = rd.get(off + i);
        if (c > 3u) { x = 1u; y = 0u; break; }
        if (comp) c = 3u - c;
        fm_step(f, c, x, y);
    }
    ox = x; oy = y;
}

// the same for a 4-bit big-endian stream (nvBowtie's read format): symbols [a, a + cnt) (1 <= cnt <= 16) squeezed to 2 bits each
// in the top 2*cnt bits of the result; `has_n` is set when one of them is > 3
__host__ __device__ __forceinline__ uint32_t squeeze_nibbles(uint32_t x)      // 8 nibbles -> 16 bits (the low 2 bits of each)
{
    uint32_t t = x & 0x33333333u;
    t = (t | (t >> 2)) & 0x0F0F0F0Fu;
    t = (t | (t >> 4)) & 0x00FF00FFu;
    return (t | (t >> 8)) & 0x0000FFFFu;
}
__host__ __device__ __forceinline__ uint32_t be4_window(const uint32_t* __restrict__ words, uint32_t a, uint32_t cnt, bool& has_n)
{
    const uint32_t wi = a >> 3, r = a & 7u, sh = 4u * r;
    const uint32_t nw = (r + cnt + 7u) >> 3;                          // words the window touches: 1..3
    const uint32_t w0 = words[wi];
    const uint32_t w1 = nw > 1u ? words[wi + 1u] : 0u;
    const uint32_t w2 = nw > 2u ? words[wi + 2u] : 0u;
    uint32_t hi = r ? ((w0 << sh) | (w1 >> (32u - sh))) : w0;         // symbols 0..7 of the window
    uint32_t lo = r ? ((w1 << sh) | (w2 >> (32u - sh))) : w1;         // symbols 8..15
    // symbols beyond cnt are not part of the window: clear them before the N test
    if (cnt < 8u)       { hi &= ~(0xFFFFFFFFu >> (4u * cnt)); lo = 0u; }
    else if (cnt < 16u) { lo &= (cnt == 8u) ? 0u : ~(0xFFFFFFFFu >> (4u * (cnt - 8u))); }
    has_n |= ((hi | lo) & 0xCCCCCCCCu) != 0u;
    return (squeeze_nibbles(hi) << 16) | squeeze_nibbles(lo);
}

// Text context words (one-row table entries, two-row entries' 7-symbol halves, the per-row array): the symbols before a text position pos,
// symbol pos-1 in the lowest two bits.  unread_context() puts the first `rem` (1..16) symbols of a query in the same order (its symbol
// rem-1 lowest; n_left is set when one of them is an N), and context_matches() tells whether the `cnt` (0..16) of them closest to pos
// -- the first ones a backward search would consume from the row of pos -- are the symbols before pos (context_equal: the same
// without the test that there are cnt symbols before pos).
template <int BITS, bool BE>
__host__ __device__ __forceinline__ uint32_t unread_context(const uint32_t* __restrict__ words, uint32_t off, uint32_t rem, bool& n_left)
{
    if (BITS == 2 && BE) return be2_window(words, off, rem) >> (32u - 2u * rem);
    if (BITS == 4 && BE) return be4_window(words, off, rem, n_left) >> (32u - 2u * rem);
    SymReader<BITS, BE> rd(words);
    uint32_t qw = 0u;
    for (uint32_t i = 0; i < rem; ++i) { const uint32_t c = rd.get(off + i); n_left |= (c > 3u); qw = (qw << 2) | (c & 3u); }
    return qw;
}
__host__ __device__ __forceinline__ bool context_equal(uint32_t qw, uint32_t ctx, uint32_t cnt)
{
    const uint32_t mask = cnt >= 16u ? 0xFFFFFFFFu : ((1u << (2u * cnt)) - 1u);
    return ((qw ^ ctx) & mask) == 0u;
}
__host__ __device__ __forceinline__ bool context_matches(uint32_t qw, uint32_t ctx, uint32_t pos, uint32_t cnt)
{
    return pos != 0xFFFFFFFFu && pos >= cnt && context_equal(qw, ctx, cnt);
}

// the widest k-mer range that the per-row array resolves: its rows are read with one gather each, all issued together
constexpr uint32_t FM_ROWS_MAX = 8;

// match() + locate() of one query in one pass, for callers that only need the hit POSITIONS of narrow ranges (the per-read
// seed + extend path): as soon as the range is a single row (x == y) and the index keeps the full suffix array, the remaining
// LF steps are replaced by one SA gather and a comparison of the not-yet-consumed symbols with the text itself:
//     LF from a single row x with symbol c is non-empty  <=>  bwt[x] == c  <=>  text[SA[x] - 1] == c   (and then SA[x'] = SA[x] - 1),
// so `rem` further steps succeed  <=>  text[SA[x] - rem, SA[x]) == the rem symbols still to consume, and the located position is
// SA[x] - rem -- exactly what locate(match(p)) returns for a single-row result (the `$` row has SA = 0 and fails, as its LF step
// does).  Returns FM_EMPTY, FM_RANGE (general inclusive range in (x, y); caller locates), or FM_LOCATED (single hit at text
// position x).  Backward order only (flags == 0); symbols > 3 never match.
// MODE (the seed-match stage splits its seeds by how many dependent gathers they need, so that a warp does not wait on its slowest
// lane): FM_WHOLE = everything in one call;  FM_DEFER = stop after the table look-up when the k-mer occurs three or more times (or
// twice, with both occurrences spelling the whole query; with a wide table, only when the entry's contexts do not decide the seed: more
// than 8 rows, a repeat of the whole query, a survivor isolated only by the last step, more unread symbols than the entry's contexts
// hold, an N) and
// return FM_DEFERRED with the range reached so far in (ox, oy);
// FM_RESUME = continue such a query: (ox, oy) hold that range on entry, the first ktab_k steps are taken as done ((0, n) = none).
enum { FM_EMPTY = 0, FM_RANGE = 1, FM_LOCATED = 2, FM_DEFERRED = 3 };
enum { FM_WHOLE = 0, FM_DEFER = 1, FM_RESUME = 2 };
template <int BITS, bool BE, int MODE = FM_WHOLE>
__host__ __device__ __forceinline__ uint32_t fm_match_locate_one(const FmIndex& f, const uint32_t* __restrict__ genome,
                                                                 const uint32_t* __restrict__ words, uint32_t off, uint32_t len,
                                                                 uint32_t& ox, uint32_t& oy)
{
    SymReader<BITS, BE> rd(words);
    uint32_t x = 0, y = f.n, s = 0;
    uint32_t known_pos = 0u, known_pos2 = 0u, ctx2 = 0u; bool have_pos = false, have_two = false, two_ctx = false;
    uint4 e = make_uint4(0u, 0u, 0u, 0u), e_hi = make_uint4(0u, 0u, 0u, 0u);     // the table entry (e_hi: second half of a wide one)
    if (MODE == FM_RESUME) { x = ox; y = oy; s = (x == 0u && y == f.n) ? 0u : f.ktab_k; }   // (0, n): deferred before any step (no look-up: an N, a short query)
    if (MODE != FM_RESUME && f.ktab_k && len >= f.ktab_k) {
        uint32_t u = 0; bool has_n = false;
        if (BITS == 2 && BE) {
            // the table index IS the big-endian bit pattern of the last k symbols: one funnel shift instead of k symbol reads
            u = be2_window(words, off + len - f.ktab_k, f.ktab_k) >> (32u - 2u * f.ktab_k);
        } else if (BITS == 4 && BE) {
            u = be4_window(words, off + len - f.ktab_k, f.ktab_k, has_n) >> (32u - 2u * f.ktab_k);
        } else {
            for (uint32_t j = 0; j < f.ktab_k; ++j) {
                const uint32_t c = rd.get(off + len - 1u - j);
                has_n |= (c > 3u);
                u |= (c & 3u) << (2u * j);
            }
        }
        if (!has_n) {
            if (f.ktab_located) {                       // the entry of a single-row k-mer carries SA[x]: no SA gather below
                gather_ktab_entry(f, u, e, e_hi);
                x = e.x; y = e.y; known_pos = e.z; known_pos2 = e.w;
                if (ktab_two_row_marker(f, y)) { ctx2 = y; y = x + 1u; two_ctx = true; }
                have_pos = (x == y); have_two = (y == x + 1u);
            } else {
                const uint2 r = gather_u2(f.ktab + u);
                x = r.x; y = r.y;
            }
            s = f.ktab_k;
        }
    }
    const bool full_sa = (f.sa_shift == 0u) && genome != nullptr;
    // does text[pos - rem, pos) equal the first `rem` (not yet consumed) symbols of the query?  (pos = SA of the row reached so far)
    auto prefix_matches = [&](const uint32_t pos, const uint32_t rem) -> bool {
        if (pos == 0xFFFFFFFFu || pos < rem) return false;
        const uint32_t p0 = pos - rem;
        bool same = true;
        if (BITS == 2 && BE) {
            // both sides are 2-bit big-endian streams: compare up to 16 symbols per step as bit patterns
            for (uint32_t i = 0; i < rem; i += 16u) {
                const uint32_t cnt = rem - i < 16u ? rem - i : 16u;
                same &= ((be2_window(words, off + i, cnt) ^ be2_window(genome, p0 + i, cnt)) >> (32u - 2u * cnt)) == 0u;
            }
        } else if (BITS == 4 && BE) {
            bool n_left = false;                                             // an N among the unread symbols matches nothing
            for (uint32_t i = 0; i < rem; i += 16u) {
                const uint32_t cnt = rem - i < 16u ? rem - i : 16u;
                same &= ((be4_window(words, off + i, cnt, n_left) ^ be2_window(genome, p0 + i, cnt)) >> (32u - 2u * cnt)) == 0u;
            }
            same &= !n_left;
        } else {
            SymReader<2, true> tr(genome);
            for (uint32_t i = 0; i < rem; ++i) same &= (rd.get(off + i) == tr.get(p0 + i));
        }
        return same;
    };
    if (have_two && full_sa && s < len) {
        // a k-mer with exactly two occurrences: both candidates are checked against the text (two independent reads) instead of
        // walking the range on; exactly one survivor = the single row the remaining LF steps would have reached, none = empty,
        // both = a genuine repeat of the whole query: that one takes the general path below
        const uint32_t rem = len - s;
        bool m0, m1;
        if (two_ctx && rem <= 7u) {
            // both candidates' preceding symbols came with the entry: no read of the text
            bool n_left = false;
            const uint32_t qw = unread_context<BITS, BE>(words, off, rem, n_left);
            m0 = !n_left && context_matches(qw, ctx2, known_pos, rem);
            m1 = !n_left && context_matches(qw, ctx2 >> 14, known_pos2, rem);
        } else {
            m0 = prefix_matches(known_pos, rem); m1 = prefix_matches(known_pos2, rem);
        }
        if (!m0 && !m1) return FM_EMPTY;
        if (m0 != m1) { ox = (m0 ? known_pos : known_pos2) - rem; oy = 0xFFFFFFFFu; return FM_LOCATED; }
    }
    if (MODE != FM_RESUME && f.ktab_wide && full_sa && s == f.ktab_k && s < len && y - x >= 2u && y - x < KTAB_WIDE_ROWS) {
        // a k-mer with 3..8 occurrences on a wide table: the rule of the per-row array below, decided on the contexts that came with the
        // look-up.  They are 16 symbols long for 3 rows and 8 for 4..8, so the unread symbols are compared over min(rem, width) of them:
        // no survivor = empty (exact: a longer remainder or a short context near the text start can only add survivors); with rem <= width,
        // one survivor that is also the only row matching the rem - 1 closest symbols = located, at its SA value from the entry (3 or 4
        // rows) or from the full suffix array (5 to 8 rows: one more gather).  As with the per-row array, the contexts are compared
        // without the position test, which can only add survivors, and the single survivor's SA is tested after.  Anything else is
        // deferred or walked as without the wide half.
        const uint32_t rem = len - s, cnt = rem < 16u ? rem : 16u;
        const bool three = (y - x == 2u);
        const uint32_t width = three ? 16u : 8u, wc = cnt < width ? cnt : width;
        bool n_left = false;
        const uint32_t qw = unread_context<BITS, BE>(words, off + rem - cnt, cnt, n_left);     // the cnt unread symbols closest to the k-mer
        if (!n_left) {
            uint32_t full = 0u, near = 0u, hit = 0u;
#pragma unroll
            for (uint32_t i = 0; i < KTAB_WIDE_ROWS; ++i) {
                if (i > y - x) continue;
                const uint32_t c = ktab_wide_context(e, e_hi, three, i);
                if (context_equal(qw, c, wc)) { ++full; hit = i; }
                near += context_equal(qw, c, wc - 1u) ? 1u : 0u;
            }
            if (full == 0u) return FM_EMPTY;
            if (full == 1u && near == 1u && rem <= width) {
                const uint32_t pos = y - x <= 3u ? ktab_wide_sa(e, e_hi, three, hit) : gather_u32(f.ssa + x + hit);
                if (pos == 0xFFFFFFFFu || pos < rem) return FM_EMPTY;
                ox = pos - rem; oy = 0xFFFFFFFFu;
                return FM_LOCATED;
            }
        }
    }
    if (MODE != FM_DEFER && f.rows && full_sa && s == f.ktab_k && s < len && y - x >= 2u && y - x < FM_ROWS_MAX && len - s <= 16u) {
        // a k-mer with 3..FM_ROWS_MAX occurrences, on an index with the per-row array: the rows' contexts are compared with the unread
        // symbols instead of walking the range on.  Row r survives the rem remaining LF steps <=> the rem symbols before SA[r] are the
        // unread ones, and it is still in the range after j steps <=> the j symbols before SA[r] match.  The walk stops at the first
        // step where one row is left and locates it there; when that happens only after the last step it returns the one-row RANGE
        // instead.  So: no survivor = empty; one survivor that is also the only row matching the rem - 1 symbols closest to it =
        // located at SA[r] - rem; anything else (a repeat of the whole query, a range narrowed to one row by its last step, an N
        // among the unread symbols) takes the walk below, which is unchanged.
        // Only the context words are gathered first (one register per row in flight, not two), so the position test of
        // context_matches is left out: that can only add rows (a row with SA[r] < 16 has fewer context symbols), never drop one.
        // An empty set stays exact, two or more take the walk, and a single survivor's SA[r] -- in the sector just read -- is
        // checked after.
        const uint32_t rem = len - s;
        bool n_left = false;
        const uint32_t qw = unread_context<BITS, BE>(words, off, rem, n_left);
        if (!n_left) {
            const uint32_t* ctx = (const uint32_t*)(f.rows + x) + 1;
            uint32_t c[FM_ROWS_MAX];
#pragma unroll
            for (uint32_t i = 0; i < FM_ROWS_MAX; ++i) c[i] = (i <= y - x) ? gather_u32(ctx + 2u * i) : 0u;
            uint32_t full = 0u, near = 0u, hit = 0u;
#pragma unroll
            for (uint32_t i = 0; i < FM_ROWS_MAX; ++i) {
                if (i > y - x) continue;
                if (context_equal(qw, c[i], rem)) { ++full; hit = i; }
                near += context_equal(qw, c[i], rem - 1u) ? 1u : 0u;
            }
            if (full == 0u) return FM_EMPTY;
            if (full == 1u && near == 1u) {
                const uint32_t pos = gather_u32((const uint32_t*)(f.rows + x + hit));
                if (pos == 0xFFFFFFFFu || pos < rem) return FM_EMPTY;
                ox = pos - rem; oy = 0xFFFFFFFFu;
                return FM_LOCATED;
            }
        }
    }
    if (MODE == FM_DEFER && s < len && x < y) { ox = x; oy = y; return FM_DEFERRED; }
    for (; s < len && x <= y; ++s) {
        if (full_sa && x == y) {
            const uint32_t rem = len - s;                 // symbols [0, rem) of the query are still to be consumed
            // (have_pos can only be set on the first pass: a single-row range returns from this branch)
            const uint32_t pos = have_pos ? known_pos : gather_u32(f.ssa + x);
            if (have_pos && f.ktab_located == 2u && rem <= 16u) {
                // the entry also carries the 16 text symbols before SA[x] (symbol SA[x]-1 in the lowest bits): the comparison needs
                // no read of the text at all -- the look-up was this seed's only gather
                bool n_left = false;
                const uint32_t qw = unread_context<BITS, BE>(words, off, rem, n_left);
                if (n_left || !context_matches(qw, known_pos2, pos, rem)) return FM_EMPTY;
                ox = pos - rem; oy = 0xFFFFFFFFu;
                return FM_LOCATED;
            }
            if (!prefix_matches(pos, rem)) return FM_EMPTY;
            ox = pos - rem; oy = 0xFFFFFFFFu;
            return FM_LOCATED;
        }
        if (MODE == FM_DEFER) { ox = x; oy = y; return FM_DEFERRED; }     // (a single row without the full suffix array: walks on later)
        const uint32_t c = rd.get(off + len - 1u - s);
        if (c > 3u) return FM_EMPTY;
        fm_step(f, c, x, y);
    }
    if (x > y) return FM_EMPTY;
    ox = x; oy = y;
    return FM_RANGE;
}

// nvBowtie's map<find_exact>(query, len1, len2, ...) (nvBowtie/bowtie2/cuda/mapping_inl.h:128-220): hits that match
// exactly over the first len1 consumed symbols and carry exactly one substitution among symbols [len1, len2), plus the
// perfect match when find_exact.  Symbols are taken in CONSUMPTION order (query[i] of the reference's reader): stream
// order with NVB_MATCH_FORWARD_ORDER, reversed without; complemented with NVB_MATCH_COMPLEMENT.
// Ranges are written in the reference's push order (position ascending, substituted symbol ascending, exact last) to
// out[0..max_out); the return value counts every push (it may exceed max_out) and range_sum adds their sizes.
template <int BITS, bool BE>
__host__ __device__ inline uint32_t fm_map_approx_one(const FmIndex& f, const uint32_t* __restrict__ words,
                                                      uint32_t off, uint32_t len2, uint32_t len1, uint32_t flags, bool find_exact,
                                                      uint2* __restrict__ out, uint32_t max_out, uint32_t& range_sum)
{
    const bool fwd = (flags & NVB_MATCH_FORWARD_ORDER) != 0;
    const bool comp = (flags & NVB_MATCH_COMPLEMENT) != 0;
    SymReader<BITS, BE> rd(words);
    auto sym = [&](uint32_t i) -> uint32_t {
        const uint32_t c = rd.get(off + (fwd ? i : (len2 - 1u - i)));
        return (comp && c < 4u) ? 3u - c : c;
    };
    range_sum = 0;
    uint32_t n_out = 0;
    if (len1 > len2) len1 = len2;
    // an N inside the exact region, or a second N, rules the seed out; a single N later stops exact matching there
    uint32_t n_pos = 0, n_cnt = 0;
    for (uint32_t i = 0; i < len2; ++i) {
        if (sym(i) > 3u) {
            if (i < len1 || n_cnt) return 0u;
            n_pos = i; ++n_cnt;
        }
    }
    if (n_cnt) len1 = n_pos;

    uint32_t bx = 0, by = f.n;
    for (uint32_t i = 0; i < len1 && bx <= by; ++i) fm_step(f, sym(i), bx, by);

    for (uint32_t i = len1; i < len2 && bx <= by; ++i) {
        const uint32_t c = sym(i);
        const uint4 lo = fm_rank4(f, bx - 1u), hi = fm_rank4(f, by);
        const uint32_t los[4] = { lo.x, lo.y, lo.z, lo.w }, his[4] = { hi.x, hi.y, hi.z, hi.w };
#pragma unroll
        for (uint32_t sub = 0; sub < 4; ++sub) {
            if (sub != c && his[sub] > los[sub]) {
                uint32_t x = f.l2(sub) + los[sub] + 1u, y = f.l2(sub) + his[sub];
                for (uint32_t k = i + 1u; k < len2 && x <= y; ++k) {
                    const uint32_t ck = sym(k);
                    if (ck > 3u) { x = 1u; y = 0u; break; }
                    fm_step(f, ck, x, y);
                }
                if (x <= y) {
                    if (n_out < max_out) out[n_out] = make_uint2(x, y);
                    ++n_out; range_sum += y - x + 1u;
                }
            }
        }
        if (c < 4u) { bx = f.l2(c) + los[c] + 1u; by = f.l2(c) + his[c]; }
        else { bx = 1u; by = 0u; break; }
    }
    if (find_exact && bx <= by) {
        if (n_out < max_out) out[n_out] = make_uint2(bx, by);
        ++n_out; range_sum += by - bx + 1u;
    }
    return n_out;
}

// locate(fmi, row)
__host__ __device__ __forceinline__ uint32_t fm_locate_one(const FmIndex& f, uint32_t row) {
    uint32_t j = row, t = 0;
    while ((j & f.sa_mask) != 0u) {
        if (j != f.primary) {
            const uint32_t k = j < f.primary ? j : j - 1u;
            const FmBlock b = load_block(f.blocks, k >> 6);
            const uint32_t c = block_symbol(b, k & 63u);
            j = f.l2(c) + block_rank(b, k & 63u, c);
        } else {
            j = 0u;
        }
        ++t;
    }
    return gather_u32(f.ssa + (j >> f.sa_shift)) + t;
}

} // namespace nvb
