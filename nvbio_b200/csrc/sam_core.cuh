// sam_core.cuh -- per-record routines of nvb_sam_format (sam.cu) that the tests also run on the host (tests/host/sam_harness.cu): the
// validity and exact SAM line length of a BAM record (sam_line_size), and the composition of its line (sam_compose).  The rule is stated
// in include/nvbio_b200.h.
#pragma once
#include "common.cuh"

namespace nvb {

constexpr uint32_t SAM_FIXED = 36u;                  // block_size + the 32-byte core of a record

__host__ __device__ __forceinline__ uint32_t sam_ld32(const uint8_t* p)
{
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}

// decimal digits of x; of v with its sign
__host__ __device__ __forceinline__ uint32_t sam_udigits(uint32_t x)
{
    return 1u + (x >= 10u) + (x >= 100u) + (x >= 1000u) + (x >= 10000u) + (x >= 100000u) + (x >= 1000000u) + (x >= 10000000u) +
           (x >= 100000000u) + (x >= 1000000000u);
}
__host__ __device__ __forceinline__ uint32_t sam_sdigits(int32_t v) { return v < 0 ? 1u + sam_udigits(0u - (uint32_t)v) : sam_udigits((uint32_t)v); }

// x in nd digits at p; v with its sign (kputw / kputuw); both return the byte after the number
__host__ __device__ __forceinline__ char* sam_put_u(char* p, uint32_t x, uint32_t nd)
{
    for (uint32_t i = nd; i-- > 0u;) { p[i] = (char)('0' + x % 10u); x /= 10u; }
    return p + nd;
}
__host__ __device__ __forceinline__ char* sam_put_s(char* p, int32_t v)
{
    if (v < 0) { *p++ = '-'; const uint32_t x = 0u - (uint32_t)v; return sam_put_u(p, x, sam_udigits(x)); }
    return sam_put_u(p, (uint32_t)v, sam_udigits((uint32_t)v));
}

// the fixed fields of a record (r = its first byte, block_size's)
struct SamCore {
    int32_t  ref, pos, nref, npos, tlen;
    uint32_t mapq, l_name, flag, nc, l_seq;
};
__host__ __device__ __forceinline__ SamCore sam_core(const uint8_t* r)
{
    SamCore c;
    c.ref = (int32_t)sam_ld32(r + 4); c.pos = (int32_t)sam_ld32(r + 8);
    const uint32_t w2 = sam_ld32(r + 12), w3 = sam_ld32(r + 16);
    c.l_name = w2 & 0xFFu; c.mapq = (w2 >> 8) & 0xFFu;
    c.flag = w3 >> 16; c.nc = w3 & 0xFFFFu;
    c.l_seq = sam_ld32(r + 20);
    c.nref = (int32_t)sam_ld32(r + 24); c.npos = (int32_t)sam_ld32(r + 28); c.tlen = (int32_t)sam_ld32(r + 32);
    return c;
}

// POS + 1 / PNEXT + 1 as htslib's int arithmetic gives them
__host__ __device__ __forceinline__ int32_t sam_plus1(int32_t v) { return (int32_t)((uint32_t)v + 1u); }

__host__ __device__ __forceinline__ uint32_t sam_name_len(const uint32_t* off, int32_t j) { return off[j + 1] - off[j]; }

// text bytes of the header fields after QNAME: "\tFLAG\tRNAME\tPOS\tMAPQ\t"
__host__ __device__ __forceinline__ uint32_t sam_head_len(const SamCore& c, const uint32_t* ref_off)
{
    return 5u + sam_udigits(c.flag) + (c.ref < 0 ? 1u : sam_name_len(ref_off, c.ref)) + sam_sdigits(sam_plus1(c.pos)) + sam_udigits(c.mapq);
}
// text bytes of "RNEXT\tPNEXT\tTLEN\t"
__host__ __device__ __forceinline__ uint32_t sam_mate_len(const SamCore& c, const uint32_t* ref_off)
{
    return 3u + (c.nref < 0 || c.nref == c.ref ? 1u : sam_name_len(ref_off, c.nref)) + sam_sdigits(sam_plus1(c.npos)) + sam_sdigits(c.tlen);
}

// the integer value of a tag of type t (one of c C s S i I) at v, as sign and magnitude; its bytes (0: not an integer type)
__host__ __device__ __forceinline__ uint32_t sam_int_bytes(uint8_t t)
{
    return (t == 'c' || t == 'C') ? 1u : ((t == 's' || t == 'S') ? 2u : ((t == 'i' || t == 'I') ? 4u : 0u));
}
__host__ __device__ __forceinline__ uint32_t sam_int_value(uint8_t t, const uint8_t* v, bool& neg)
{
    int32_t s;
    switch (t) {
    case 'C': neg = false; return v[0];
    case 'S': neg = false; return (uint32_t)v[0] | (uint32_t)v[1] << 8;
    case 'I': neg = false; return sam_ld32(v);
    case 'c': s = (int8_t)v[0]; break;
    case 's': s = (int16_t)((uint32_t)v[0] | (uint32_t)v[1] << 8); break;
    default:  s = (int32_t)sam_ld32(v); break;
    }
    neg = s < 0;
    return neg ? 0u - (uint32_t)s : (uint32_t)s;
}

// The validity and the line length ('\n' included) of the record at r, `extent` bytes; 0 when it is rejected.
__host__ __device__ inline uint64_t sam_line_size(const uint8_t* r, uint64_t extent, uint32_t n_refs, const uint32_t* ref_off)
{
    if (extent < SAM_FIXED || (uint64_t)sam_ld32(r) + 4u != extent) return 0u;
    const SamCore c = sam_core(r);
    if (c.ref < -1 || c.ref >= (int64_t)n_refs || c.nref < -1 || c.nref >= (int64_t)n_refs) return 0u;
    const uint64_t cg = SAM_FIXED + c.l_name, sq = cg + 4u * (uint64_t)c.nc, ql = sq + ((uint64_t)c.l_seq + 1u) / 2u, aux = ql + c.l_seq;
    if (c.l_name < 2u || aux > extent || r[cg - 1u] != 0u) return 0u;
    uint64_t size = (c.l_name - 1u) + sam_head_len(c, ref_off) + sam_mate_len(c, ref_off) + 1u;
    uint32_t cig = 0u;
    for (uint32_t i = 0; i < c.nc; ++i) {
        const uint32_t op = sam_ld32(r + cg + 4u * i);
        if ((op & 15u) > 8u) return 0u;
        cig += sam_udigits(op >> 4) + 1u;
    }
    size += c.nc ? cig : 1u;
    size += c.l_seq ? (uint64_t)c.l_seq + 1u + (r[ql] == 0xFFu ? 1u : c.l_seq) : 3u;
    uint64_t p = aux;
    while (extent - p >= 4u) {
        const uint8_t t = r[p + 2u];
        p += 3u;
        if (t == 'Z') {
            const uint64_t z = p;
            while (p < extent && r[p]) ++p;
            if (p >= extent) return 0u;
            size += 6u + (p - z);
            ++p;
            continue;
        }
        const uint32_t nb = sam_int_bytes(t);
        if (!nb || p + nb > extent) return 0u;
        bool neg;
        const uint32_t m = sam_int_value(t, r + p, neg);
        size += 6u + neg + sam_udigits(m);
        p += nb;
    }
    if (p != extent) return 0u;
    return size + 1u;
}

// Exclusive sum over the lanes of f(lane), and the total.  The device runs it as a warp scan (all 32 lanes, nl = 32); the host, whose
// lanes run one after another, sums f over the lanes before `lane`.
template <typename F>
__host__ __device__ __forceinline__ uint32_t sam_lanes_exclusive_sum(F f, uint32_t lane, uint32_t nl, uint32_t& total)
{
#ifdef __CUDA_ARCH__
    const uint32_t v = f(lane);
    uint32_t x = v;
    for (uint32_t o = 1u; o < 32u; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    total = __shfl_sync(0xFFFFFFFFu, x, 31);
    return x - v;
#else
    uint32_t s = 0u, t = 0u;
    for (uint32_t i = 0; i < nl; ++i) {
        const uint32_t w = f(i);
        if (i < lane) s += w;
        t += w;
    }
    total = t;
    return s;
#endif
}

// Compose the line of a valid record r (size = sam_line_size > 0) at dst.  The work is split over nl lanes, lane `lane` writing its
// share: the name, SEQ and QUAL strided over the lanes, the CIGAR ops placed by a prefix sum of their text lengths, the fixed fields by
// lanes 0 and 1, tag j by lane j % nl.  Every byte is written by exactly one lane, so lanes 0 .. nl - 1 run one after another (the host)
// give what a warp gives; on the device the whole warp calls it (nl = 32).
__host__ __device__ inline void sam_compose(const uint8_t* __restrict__ r, uint64_t size, const char* __restrict__ ref_names,
                                            const uint32_t* __restrict__ ref_off, char* __restrict__ dst, uint32_t lane, uint32_t nl)
{
    const SamCore c = sam_core(r);
    const uint8_t* name = r + SAM_FIXED;
    char* p = dst;
    for (uint32_t i = lane; i + 1u < c.l_name; i += nl) p[i] = (char)name[i];
    p += c.l_name - 1u;
    if (lane == 0u) {                                 // \tFLAG\tRNAME\tPOS\tMAPQ\t
        char* q = p;
        *q++ = '\t';
        q = sam_put_u(q, c.flag, sam_udigits(c.flag));
        *q++ = '\t';
        if (c.ref < 0) *q++ = '*';
        else for (uint32_t i = ref_off[c.ref]; i < ref_off[c.ref + 1]; ++i) *q++ = ref_names[i];
        *q++ = '\t';
        q = sam_put_s(q, sam_plus1(c.pos));
        *q++ = '\t';
        q = sam_put_u(q, c.mapq, sam_udigits(c.mapq));
        *q = '\t';
    }
    p += sam_head_len(c, ref_off);
    const uint8_t* cg = name + c.l_name;
    uint32_t cig = 0u;
    if (c.nc == 0u) {
        if (lane == 0u) p[0] = '*';
        cig = 1u;
    }
    for (uint32_t c0 = 0; c0 < c.nc; c0 += nl) {
        uint32_t total;
        const uint32_t pre = sam_lanes_exclusive_sum([&](uint32_t l) { return c0 + l < c.nc ? sam_udigits(sam_ld32(cg + 4u * (c0 + l)) >> 4) + 1u : 0u; },
                                                     lane, nl, total);
        if (c0 + lane < c.nc) {
            const uint32_t op = sam_ld32(cg + 4u * (c0 + lane));
            char* q = sam_put_u(p + cig + pre, op >> 4, sam_udigits(op >> 4));
            *q = "MIDNSHP=X"[op & 15u];
        }
        cig += total;
    }
    p += cig;
    if (lane == 1u % nl) {                            // \tRNEXT\tPNEXT\tTLEN\t
        char* q = p;
        *q++ = '\t';
        if (c.nref < 0) *q++ = '*';
        else if (c.nref == c.ref) *q++ = '=';
        else for (uint32_t i = ref_off[c.nref]; i < ref_off[c.nref + 1]; ++i) *q++ = ref_names[i];
        *q++ = '\t';
        q = sam_put_s(q, sam_plus1(c.npos));
        *q++ = '\t';
        q = sam_put_s(q, c.tlen);
        *q = '\t';
    }
    p += 1u + sam_mate_len(c, ref_off);
    const uint8_t* seq = cg + 4u * c.nc;
    const uint8_t* qual = seq + (c.l_seq + 1u) / 2u;
    const uint32_t l = c.l_seq;
    if (l == 0u) {
        if (lane == 0u) { p[0] = '*'; p[1] = '\t'; p[2] = '*'; }
        p += 3u;
    } else {
        for (uint32_t j = lane; 2u * j < l; j += nl) {
            const uint32_t b = seq[j];
            p[2u * j] = "=ACMGRSVTWYHKDBN"[b >> 4];
            if (2u * j + 1u < l) p[2u * j + 1u] = "=ACMGRSVTWYHKDBN"[b & 15u];
        }
        p += l;
        if (lane == 0u) p[0] = '\t';
        ++p;
        if (qual[0] == 0xFFu) {
            if (lane == 0u) p[0] = '*';
            ++p;
        } else {
            for (uint32_t i = lane; i < l; i += nl) p[i] = (char)(qual[i] + 33u);
            p += l;
        }
    }
    // tags: every lane walks them; tag j is written by lane j % nl
    const uint8_t* t = qual + l;
    char* const end = dst + size - 1u;
    for (uint32_t j = 0; p < end; ++j) {
        const uint8_t type = t[2];
        const bool mine = j % nl == lane;
        if (mine) { p[0] = '\t'; p[1] = (char)t[0]; p[2] = (char)t[1]; p[3] = ':'; p[4] = type == 'Z' ? 'Z' : 'i'; p[5] = ':'; }
        p += 6;
        t += 3;
        if (type == 'Z') {
            for (; *t; ++t, ++p) if (mine) *p = (char)*t;
            ++t;
        } else {
            bool neg;
            const uint32_t m = sam_int_value(type, t, neg);
            const uint32_t nd = sam_udigits(m);
            if (mine) { if (neg) *p = '-'; sam_put_u(p + neg, m, nd); }
            p += neg + nd;
            t += sam_int_bytes(type);
        }
    }
    if (lane == 0u) *end = '\n';
}

} // namespace nvb
