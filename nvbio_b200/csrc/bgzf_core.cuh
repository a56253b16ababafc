// bgzf_core.cuh -- per-block routines of nvb_bgzf_compress (bgzf.cu) that the tests also run on the host (tests/host/bgzf_harness.cu):
// CRC-32 of a chunk and the shift that combines chunk CRCs, the match rule of one position, length-limited Huffman code lengths
// (package-merge), canonical codes, the run-length coded header of a dynamic deflate block, the bits of one token and the member's
// header / footer bytes.  Written from RFC 1951 (deflate), RFC 1952 (gzip) and SAMv1 section 4.1 (BGZF); the member framing is that of
// htslib's writer (contrib/htslib/bgzf.c:59 header, bgzf.c:216-240 deflate_block, htslib/bgzf.h:36-37 block sizes).
#pragma once
#include "common.cuh"
#ifndef __CUDA_ARCH__
#include <string.h>
#endif

namespace nvb {

constexpr uint32_t BGZF_BLOCK = 0xFF00u;                 // input bytes per member (BGZF_BLOCK_SIZE, bgzf.h:36)
constexpr uint32_t BGZF_HDR = 18u, BGZF_FTR = 8u;         // member header (with the BC extra field) and CRC32 + ISIZE
constexpr uint32_t BGZF_MAX_MEMBER = BGZF_HDR + 5u + BGZF_BLOCK + BGZF_FTR;    // 65,311: a stored block of a full input block
constexpr uint32_t BGZF_SLOT = 65536u;                   // temp bytes per member before compaction
constexpr uint32_t BGZF_MIN_MATCH = 3u, BGZF_MAX_MATCH = 258u, BGZF_WINDOW = 32768u;
constexpr uint32_t BGZF_TOO_FAR = 4096u;                 // a length-3 match farther than this costs more than its 3 literals
constexpr uint32_t BGZF_HASH_BITS = 14u;
constexpr uint32_t BGZF_NLIT = 286u, BGZF_NDIST = 30u, BGZF_NCL = 19u;
constexpr uint32_t BGZF_MAX_BITS = 15u, BGZF_MAX_CL_BITS = 7u;
constexpr uint32_t BGZF_PM_ITEMS = 2u * BGZF_NLIT;       // package-merge list length bound (2m - 2 items are kept)
constexpr uint32_t CRC32_POLY = 0xEDB88320u;             // x^32 + x^26 + ... + 1, bit-reflected (RFC 1952 section 8)

__host__ __device__ __forceinline__ uint32_t bgzf_log2(uint32_t x)     // floor(log2(x)), x > 0
{
#ifdef __CUDA_ARCH__
    return 31u - (uint32_t)__clz(x);
#else
    return 31u - (uint32_t)__builtin_clz(x);
#endif
}
__host__ __device__ __forceinline__ uint32_t bgzf_ctz(uint32_t x)      // x > 0
{
#ifdef __CUDA_ARCH__
    return (uint32_t)__ffs(x) - 1u;
#else
    return (uint32_t)__builtin_ctz(x);
#endif
}
// the low n bits of x in reverse order (Huffman codes are sent most significant bit first, everything else least significant first)
__host__ __device__ __forceinline__ uint32_t bgzf_rev(uint32_t x, uint32_t n)
{
#ifdef __CUDA_ARCH__
    return __brev(x) >> (32u - n);
#else
    uint32_t r = 0u;
    for (uint32_t i = 0; i < n; ++i) r |= ((x >> i) & 1u) << (n - 1u - i);
    return r;
#endif
}
__host__ __device__ __forceinline__ void bgzf_or(uint32_t* w, uint32_t v)
{
#ifdef __CUDA_ARCH__
    atomicOr(w, v);
#else
    *w |= v;
#endif
}
// OR the low n (<= 32) bits of v into the little-endian bit stream `words` at bit `pos`; the stream is zeroed beforehand
__host__ __device__ __forceinline__ void put_bits(uint32_t* words, uint32_t pos, uint32_t v, uint32_t n)
{
    if (n == 0u) return;
    const uint32_t w = pos >> 5, s = pos & 31u;
    bgzf_or(words + w, v << s);
    if (s + n > 32u) bgzf_or(words + w + 1u, v >> (32u - s));
}

// ---------------------------------------------------------------------------------------------
// CRC-32.  The register is linear in its input: the register after A || B is shift(register after A, |B|) ^ (register of B from 0),
// where shift multiplies by x^(8 |B|) modulo the polynomial.  A block's CRC is the XOR of its chunks' shifted zero-start registers.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t crc32_table_entry(uint32_t b)       // register of byte b from 0
{
    uint32_t c = b;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (CRC32_POLY & (0u - (c & 1u)));
    return c;
}
__host__ __device__ __forceinline__ uint32_t crc32_raw(const uint32_t* __restrict__ table, const uint8_t* p, uint32_t n, uint32_t c)
{
    for (uint32_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
    return c;
}
// a * b modulo the CRC polynomial, both bit-reflected (bit 31 = x^0)
__host__ __device__ __forceinline__ uint32_t gf2_mulmod(uint32_t a, uint32_t b)
{
    uint32_t r = 0u;
    for (int i = 0; i < 32; ++i) {                           // b = b * x^i
        r ^= b & (0u - ((a >> (31 - i)) & 1u));
        b = (b >> 1) ^ (CRC32_POLY & (0u - (b & 1u)));
    }
    return r;
}
// register c followed by n zero bytes: c * x^(8n)
__host__ __device__ __forceinline__ uint32_t crc32_shift(uint32_t c, uint64_t n)
{
    uint32_t x = 0x00800000u;                                // x^8
    for (; n; n >>= 1) {
        if (n & 1u) c = gf2_mulmod(c, x);
        x = gf2_mulmod(x, x);
    }
    return c;
}

// ---------------------------------------------------------------------------------------------
// Symbols of RFC 1951 section 3.2.5
// ---------------------------------------------------------------------------------------------
// literal/length symbol of a match length 3..258, its extra-bit count and value
__host__ __device__ __forceinline__ void len_sym(uint32_t len, uint32_t& sym, uint32_t& nx, uint32_t& x)
{
    const uint32_t l = len - 3u;
    if (l < 8u)          { sym = 257u + l; nx = 0u; x = 0u; }
    else if (l == 255u)  { sym = 285u; nx = 0u; x = 0u; }
    else { const uint32_t e = bgzf_log2(l) - 2u; sym = 257u + 4u * (e + 1u) + ((l >> e) - 4u); nx = e; x = l & ((1u << e) - 1u); }
}
// distance symbol of a distance 1..32768, its extra-bit count and value
__host__ __device__ __forceinline__ void dist_sym(uint32_t dist, uint32_t& sym, uint32_t& nx, uint32_t& x)
{
    const uint32_t d = dist - 1u;
    if (d < 4u) { sym = d; nx = 0u; x = 0u; }
    else { const uint32_t e = bgzf_log2(d) - 1u; sym = 2u * (e + 1u) + ((d >> e) & 1u); nx = e; x = d & ((1u << e) - 1u); }
}
// the order in which the code-length code's lengths are sent: 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15
__host__ __device__ __forceinline__ uint32_t cl_order(uint32_t i)
{
    if (i < 3u) return 16u + i;
    if (i == 3u) return 0u;
    const uint32_t j = i - 4u;
    return (j & 1u) ? 7u - (j >> 1) : 8u + (j >> 1);
}

// ---------------------------------------------------------------------------------------------
// Match finding.  Each position looks up one hash-table candidate (the latest earlier position with the same 4-byte prefix hash,
// stored as position + 1) and distance 1, and keeps the longer match (distance 1 on ties).
// ---------------------------------------------------------------------------------------------
// 4 bytes at s[p], little-endian; s is 4-byte aligned and readable up to s[p + 7]
__host__ __device__ __forceinline__ uint32_t load32(const uint8_t* s, uint32_t p)
{
#ifdef __CUDA_ARCH__
    const uint32_t* w = (const uint32_t*)s + (p >> 2);
    return __funnelshift_r(w[0], w[1], (p & 3u) * 8u);
#else
    uint32_t v; memcpy(&v, s + p, 4); return v;
#endif
}
__host__ __device__ __forceinline__ uint32_t bgzf_hash(const uint8_t* s, uint32_t p)
{
    return (load32(s, p) * 2654435761u) >> (32u - BGZF_HASH_BITS);
}
// common prefix of s[p..] and s[q..], at most maxl bytes
__host__ __device__ __forceinline__ uint32_t match_len(const uint8_t* s, uint32_t p, uint32_t q, uint32_t maxl)
{
    uint32_t l = 0u;
    for (; l + 4u <= maxl; l += 4u) {
        const uint32_t x = load32(s, p + l) ^ load32(s, q + l);
        if (x) return l + (bgzf_ctz(x) >> 3);
    }
    while (l < maxl && s[p + l] == s[q + l]) ++l;
    return l;
}
// the match the parse takes at p of an n-byte block: (length << 16) | (distance - 1), or 0 (a literal).  cand: the table entry
__host__ __device__ __forceinline__ uint32_t find_match(const uint8_t* s, uint32_t n, uint32_t p, uint32_t cand)
{
    const uint32_t maxl = n - p < BGZF_MAX_MATCH ? n - p : BGZF_MAX_MATCH;
    if (p == 0u || maxl < BGZF_MIN_MATCH) return 0u;
    uint32_t best = match_len(s, p, p - 1u, maxl), dist = 1u;
    if (cand != 0u && cand < p && p - (cand - 1u) <= BGZF_WINDOW) {
        const uint32_t l = match_len(s, p, cand - 1u, maxl);
        if (l > best) { best = l; dist = p - (cand - 1u); }
    }
    if (best < BGZF_MIN_MATCH || (best == BGZF_MIN_MATCH && dist > BGZF_TOO_FAR)) return 0u;
    return (best << 16) | (dist - 1u);
}

// ---------------------------------------------------------------------------------------------
// Huffman codes
// ---------------------------------------------------------------------------------------------
// scratch of one length-limited code construction (shared memory on the device)
struct BgzfPm {
    uint32_t w[BGZF_NLIT];                  // weights of the used symbols in (frequency, symbol) order
    uint16_t sym[BGZF_NLIT];
    uint32_t wa[BGZF_PM_ITEMS], wb[BGZF_PM_ITEMS];
    uint8_t  leaf[BGZF_MAX_BITS - 1u][BGZF_PM_ITEMS];   // per level above the deepest: item k is a leaf
    uint32_t cnt[BGZF_MAX_BITS + 1u], next[BGZF_MAX_BITS + 1u];
};

// a code needs two used symbols to be complete: give frequency 1 to the lowest unused symbols until two are used (the extra code is
// never sent).  Returns the number of used symbols.
__host__ __device__ __forceinline__ uint32_t bump_used(uint32_t* f, uint32_t n)
{
    uint32_t m = 0u;
    for (uint32_t s = 0; s < n; ++s) m += f[s] != 0u;
    for (uint32_t s = 0; s < n && m < 2u; ++s)
        if (f[s] == 0u) { f[s] = 1u; ++m; }
    return m;
}
// rank of used symbol s among the used symbols in (frequency, symbol) order
__host__ __device__ __forceinline__ uint32_t freq_rank(const uint32_t* f, uint32_t n, uint32_t s)
{
    uint32_t r = 0u;
    const uint32_t fs = f[s];
    for (uint32_t i = 0; i < n; ++i) r += f[i] != 0u && (f[i] < fs || (f[i] == fs && i < s));
    return r;
}
// Optimal code lengths of at most `limit` bits for the m >= 2 sorted weights pm.w (package-merge, Larmore and Hirschberg 1990): the
// deepest level lists the leaves; every level above merges them with the pairs of the level below, a leaf first on equal weights; the
// first 2m - 2 items of the top level are selected, and a selected package selects the first two items per package one level down.  A
// symbol's length is the number of levels that select it.  len[pm.sym[i]] is written for the used symbols only.
__host__ __device__ inline void package_merge(BgzfPm& pm, uint32_t m, uint32_t limit, uint8_t* len)
{
    const uint32_t keep = 2u * m - 2u;
    uint32_t* prev = pm.wa; uint32_t* cur = pm.wb;
    uint32_t n_prev = m;
    for (uint32_t i = 0; i < m; ++i) prev[i] = pm.w[i];
    for (uint32_t lv = limit - 1u; lv >= 1u; --lv) {                     // level lv (1 = top) from level lv + 1
        const uint32_t np = n_prev >> 1;
        uint32_t i = 0u, k = 0u, o = 0u;
        uint8_t* leaf = pm.leaf[lv - 1u];
        while (o < keep && (i < m || k < np)) {
            const bool take_leaf = k >= np || (i < m && pm.w[i] <= prev[2u * k] + prev[2u * k + 1u]);
            if (take_leaf) { cur[o] = pm.w[i++]; leaf[o++] = 1u; }
            else           { cur[o] = prev[2u * k] + prev[2u * k + 1u]; ++k; leaf[o++] = 0u; }
        }
        n_prev = o;
        uint32_t* t = prev; prev = cur; cur = t;
    }
    for (uint32_t i = 0; i < m; ++i) len[pm.sym[i]] = 0u;
    uint32_t take = keep;
    for (uint32_t lv = 1u; lv <= limit && take; ++lv) {
        uint32_t nl = take;                                              // the deepest level holds leaves only
        if (lv < limit) { nl = 0u; for (uint32_t o = 0; o < take; ++o) nl += pm.leaf[lv - 1u][o]; }
        for (uint32_t i = 0; i < nl; ++i) ++len[pm.sym[i]];
        take = 2u * (take - nl);
    }
}
// code lengths of the frequencies f[0..n) (bumped to two used symbols), serially: the host build and the small code-length code
__host__ __device__ inline void code_lengths(uint32_t* f, uint32_t n, uint32_t limit, uint8_t* len, BgzfPm& pm)
{
    const uint32_t m = bump_used(f, n);
    for (uint32_t s = 0; s < n; ++s) {
        len[s] = 0u;
        if (f[s]) { const uint32_t r = freq_rank(f, n, s); pm.sym[r] = (uint16_t)s; pm.w[r] = f[s]; }
    }
    package_merge(pm, m, limit, len);
}
// canonical codes of the lengths (RFC 1951 section 3.2.2), bit-reversed for the least-significant-first stream
__host__ __device__ inline void canonical_codes(const uint8_t* len, uint32_t n, uint16_t* code, BgzfPm& pm)
{
    for (uint32_t b = 0; b <= BGZF_MAX_BITS; ++b) pm.cnt[b] = 0u;
    for (uint32_t s = 0; s < n; ++s) ++pm.cnt[len[s]];
    pm.cnt[0] = 0u;
    uint32_t c = 0u;
    for (uint32_t b = 1; b <= BGZF_MAX_BITS; ++b) { c = (c + pm.cnt[b - 1u]) << 1; pm.next[b] = c; }
    for (uint32_t s = 0; s < n; ++s) code[s] = len[s] ? (uint16_t)bgzf_rev(pm.next[len[s]]++, len[s]) : (uint16_t)0u;
}

// the codes of one dynamic block and its header (RFC 1951 section 3.2.7)
struct BgzfCodes {
    uint8_t  lit_len[BGZF_NLIT], dist_len[BGZF_NDIST], cl_len[BGZF_NCL];
    uint16_t lit_code[BGZF_NLIT], dist_code[BGZF_NDIST], cl_code[BGZF_NCL];
    uint16_t rle[BGZF_NLIT + BGZF_NDIST];   // code-length symbols: symbol | extra value << 5
    uint32_t cl_freq[BGZF_NCL];
    uint32_t n_rle, hlit, hdist, hclen;
    uint32_t header_bits;                   // BFINAL, BTYPE and the header
};
__host__ __device__ __forceinline__ uint32_t cl_extra_bits(uint32_t sym) { return sym == 16u ? 2u : sym == 17u ? 3u : sym == 18u ? 7u : 0u; }

// with lit_len / dist_len set: canonical codes, the run-length coded lengths, the code-length code, HCLEN and the header's size
__host__ __device__ inline void plan_header(BgzfCodes& c, BgzfPm& pm)
{
    canonical_codes(c.lit_len, BGZF_NLIT, c.lit_code, pm);
    canonical_codes(c.dist_len, BGZF_NDIST, c.dist_code, pm);
    c.hlit = BGZF_NLIT;  while (c.hlit > 257u && c.lit_len[c.hlit - 1u] == 0u) --c.hlit;
    c.hdist = BGZF_NDIST; while (c.hdist > 1u && c.dist_len[c.hdist - 1u] == 0u) --c.hdist;
    // the lengths form one sequence of hlit + hdist values; runs may cross from the literal/length part to the distance part
    const uint32_t total = c.hlit + c.hdist;
    for (uint32_t s = 0; s < BGZF_NCL; ++s) c.cl_freq[s] = 0u;
    c.n_rle = 0u;
    for (uint32_t i = 0; i < total;) {
        const uint32_t v = i < c.hlit ? c.lit_len[i] : c.dist_len[i - c.hlit];
        uint32_t r = 1u;
        while (i + r < total && (i + r < c.hlit ? c.lit_len[i + r] : c.dist_len[i + r - c.hlit]) == v) ++r;
        i += r;
        if (v == 0u) {
            while (r >= 11u) { const uint32_t k = r < 138u ? r : 138u; c.rle[c.n_rle++] = (uint16_t)(18u | (k - 11u) << 5); ++c.cl_freq[18]; r -= k; }
            if (r >= 3u) { c.rle[c.n_rle++] = (uint16_t)(17u | (r - 3u) << 5); ++c.cl_freq[17]; r = 0u; }
        } else {
            c.rle[c.n_rle++] = (uint16_t)v; ++c.cl_freq[v]; --r;
            while (r >= 3u) { const uint32_t k = r < 6u ? r : 6u; c.rle[c.n_rle++] = (uint16_t)(16u | (k - 3u) << 5); ++c.cl_freq[16]; r -= k; }
        }
        for (; r; --r) { c.rle[c.n_rle++] = (uint16_t)v; ++c.cl_freq[v]; }
    }
    code_lengths(c.cl_freq, BGZF_NCL, BGZF_MAX_CL_BITS, c.cl_len, pm);
    canonical_codes(c.cl_len, BGZF_NCL, c.cl_code, pm);
    c.hclen = BGZF_NCL;
    while (c.hclen > 4u && c.cl_len[cl_order(c.hclen - 1u)] == 0u) --c.hclen;
    uint32_t bits = 3u + 5u + 5u + 4u + 3u * c.hclen;
    for (uint32_t k = 0; k < c.n_rle; ++k) { const uint32_t s = c.rle[k] & 31u; bits += c.cl_len[s] + cl_extra_bits(s); }
    c.header_bits = bits;
}
// BFINAL = 1, BTYPE = 2 and the header at bit `pos`; returns the bits written (= header_bits)
__host__ __device__ inline uint32_t write_header(uint32_t* out, uint32_t pos, const BgzfCodes& c)
{
    const uint32_t p0 = pos;
    put_bits(out, pos, 1u | 2u << 1, 3u); pos += 3u;
    put_bits(out, pos, c.hlit - 257u, 5u); pos += 5u;
    put_bits(out, pos, c.hdist - 1u, 5u); pos += 5u;
    put_bits(out, pos, c.hclen - 4u, 4u); pos += 4u;
    for (uint32_t k = 0; k < c.hclen; ++k) { put_bits(out, pos, c.cl_len[cl_order(k)], 3u); pos += 3u; }
    for (uint32_t k = 0; k < c.n_rle; ++k) {
        const uint32_t s = c.rle[k] & 31u, x = c.rle[k] >> 5, nx = cl_extra_bits(s);
        put_bits(out, pos, c.cl_code[s], c.cl_len[s]); pos += c.cl_len[s];
        put_bits(out, pos, x, nx); pos += nx;
    }
    return pos - p0;
}

// ---------------------------------------------------------------------------------------------
// Tokens of the parse.  A block's parse state: the input, the match bit of every position (mbit), the length - 3 (mlen) and distance - 1
// (dist) where it is set.
// ---------------------------------------------------------------------------------------------
struct BgzfParse {
    const uint8_t*  in;
    const uint8_t*  mlen;
    const uint32_t* mbit;
    const uint16_t* dist;
};
__host__ __device__ __forceinline__ bool is_match(const uint32_t* mbit, uint32_t p) { return (mbit[p >> 5] >> (p & 31u)) & 1u; }
// bytes the token at p covers
__host__ __device__ __forceinline__ uint32_t token_advance(const BgzfParse& v, uint32_t p) { return is_match(v.mbit, p) ? v.mlen[p] + 3u : 1u; }
// count the token at p into the histograms
__host__ __device__ __forceinline__ void count_token(const BgzfParse& v, uint32_t p, uint32_t* hlit, uint32_t* hdist)
{
    uint32_t ls = v.in[p], ds = 0u, nx, x;
    const bool m = is_match(v.mbit, p);
    if (m) { len_sym(v.mlen[p] + 3u, ls, nx, x); dist_sym(v.dist[p] + 1u, ds, nx, x); }
#ifdef __CUDA_ARCH__
    atomicAdd(hlit + ls, 1u);
    if (m) atomicAdd(hdist + ds, 1u);
#else
    ++hlit[ls];
    if (m) ++hdist[ds];
#endif
}
// the token at p: bits it takes (and, with out != NULL, written at bit pos)
__host__ __device__ __forceinline__ uint32_t put_token(const BgzfParse& v, const BgzfCodes& c, uint32_t p, uint32_t* out, uint32_t pos)
{
    if (!is_match(v.mbit, p)) {
        const uint32_t s = v.in[p];
        if (out) put_bits(out, pos, c.lit_code[s], c.lit_len[s]);
        return c.lit_len[s];
    }
    uint32_t ls, lnx, lx, ds, dnx, dx;
    len_sym(v.mlen[p] + 3u, ls, lnx, lx);
    dist_sym(v.dist[p] + 1u, ds, dnx, dx);
    const uint32_t a = c.lit_len[ls] + lnx, b = c.dist_len[ds] + dnx;
    if (out) {
        put_bits(out, pos, c.lit_code[ls] | lx << c.lit_len[ls], a);
        put_bits(out, pos + a, c.dist_code[ds] | dx << c.dist_len[ds], b);
    }
    return a + b;
}

// ---------------------------------------------------------------------------------------------
// Member framing (SAMv1 section 4.1.1, RFC 1952): byte k (k < 18) of the header of a member of `member` bytes, byte k (k < 8) of the
// footer, and byte k (k < 5) of a stored deflate block of n bytes (BFINAL = 1, BTYPE = 0, LEN, NLEN)
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint8_t member_header_byte(uint32_t k, uint32_t member)
{
    // ID1 ID2 CM FLG(FEXTRA) | MTIME(4) = 0 | XFL 0, OS 255, XLEN 6 | 'B' 'C' SLEN 2 | BSIZE = member - 1
    switch (k) {
        case 0: return 0x1Fu;  case 1: return 0x8Bu;  case 2: return 8u;  case 3: return 4u;
        case 9: return 0xFFu;  case 10: return 6u;    case 12: return 'B'; case 13: return 'C';  case 14: return 2u;
        case 16: return (uint8_t)(member - 1u);       case 17: return (uint8_t)((member - 1u) >> 8);
        default: return 0u;
    }
}
__host__ __device__ __forceinline__ uint8_t member_footer_byte(uint32_t k, uint32_t crc, uint32_t n)
{
    return (uint8_t)((k < 4u ? crc : n) >> (8u * (k & 3u)));
}
__host__ __device__ __forceinline__ uint8_t stored_header_byte(uint32_t k, uint32_t n)
{
    if (k == 0u) return 1u;
    const uint32_t v = k < 3u ? n : (~n & 0xFFFFu);
    return (uint8_t)(v >> (8u * ((k - 1u) & 1u)));
}

} // namespace nvb
