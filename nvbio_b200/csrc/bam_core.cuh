// bam_core.cuh -- per-record routines of nvb_bam_records (bam.cu) that the tests also run on the host (tests/host/bam_harness.cu):
// the placement of an alignment on the contig table, the 32-byte core of its BAM record (FLAG, MAPQ, bin, mate fields, TLEN) and its
// size, and the composition of the whole record (name, CIGAR, SEQ, QUAL, tags).
#pragma once
#include "finish_core.cuh"

namespace nvb {

constexpr uint32_t BAM_FIXED = 36u;                  // block_size + the 32-byte core of a record
constexpr uint32_t BAM_MAX_NAME = 254u;              // l_read_name is one byte and counts the NUL

// hts_reg2bin(beg, end, 14, 5) (contrib/htslib/htslib/hts.h:254-260): the smallest bin of the specification's binning index that holds
// [beg, end); the same signed arithmetic, so [-1, 0) of an unplaced record gives 4680
__host__ __device__ __forceinline__ uint32_t bam_reg2bin(int64_t beg, int64_t end)
{
    --end;
    if (beg >> 14 == end >> 14) return (uint32_t)(((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (uint32_t)(((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (uint32_t)(((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (uint32_t)(((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (uint32_t)(((1 << 3) - 1) / 7 + (beg >> 26));
    return 0u;
}

// bytes of an integer tag's value in the type htslib's SAM parser gives it: the smallest of c / s / i (negative) or C / S / I
__host__ __device__ __forceinline__ uint32_t tag_int_bytes(int64_t v)
{
    if (v < 0) return v >= -128 ? 1u : (v >= -32768 ? 2u : 4u);
    return v <= 255 ? 1u : (v <= 65535 ? 2u : 4u);
}
__host__ __device__ __forceinline__ uint32_t tag_int_type(int64_t v, uint32_t bytes)
{
    return v < 0 ? (bytes == 1u ? 'c' : (bytes == 2u ? 's' : 'i')) : (bytes == 1u ? 'C' : (bytes == 2u ? 'S' : 'I'));
}

// the inputs of nvb_bam_records as the kernels see them
struct BamIn {
    StrSet          reads;
    const uint8_t*  quals;
    const uint32_t* n_ops;
    const uint2*    begin;
    const uint8_t*  strand;
    const uint32_t* cigar;  uint32_t max_cigar; const uint32_t* n_cigar;
    const char*     md;     uint32_t max_md;    const uint32_t* md_len;
    const uint32_t* edits;
    const int32_t*  score;
    const uint8_t*  mapq;
    const int32_t*  second;
    const uint32_t* pair_flags;
    const uint32_t* contig_begin; uint32_t n_contigs;
    const char*     names;  const uint32_t* name_off;
    uint32_t        n;                              // alignments (= records); nvb_bam_records_all: record slots
    const uint4*    rec = nullptr;                  // nvb_bam_records_all: record k = (alignment or BAM_NO_ALN, read, NH, primary); else NULL
};

constexpr uint32_t BAM_NO_ALN = 0xFFFFFFFFu;        // the unmapped record of a read without a placeable alignment

// alignment of record k (paired: record 2p + m is mate m of pair p, alignment m * n / 2 + p), the index of its name and of its read in
// `reads`; mapq / second score are per alignment in nvb_bam_records and per read in nvb_bam_records_all
__host__ __device__ __forceinline__ uint32_t bam_alignment(const BamIn& in, uint32_t k)
{
    return in.rec ? in.rec[k].x : (in.pair_flags ? (k & 1u) * (in.n >> 1) + (k >> 1) : k);
}
__host__ __device__ __forceinline__ uint32_t bam_name(const BamIn& in, uint32_t k) { return in.rec ? in.rec[k].y : (in.pair_flags ? k >> 1 : k); }
__host__ __device__ __forceinline__ uint32_t bam_seq(const BamIn& in, uint32_t k) { return in.rec ? in.rec[k].y : bam_alignment(in, k); }
// XS of mapped record k (alignment a): INT32_MIN = none.  nvb_bam_records_all: the read's second score, on its primary record only
__host__ __device__ __forceinline__ int32_t bam_xs(const BamIn& in, uint32_t k, uint32_t a)
{
    if (!in.second) return INT32_MIN;
    if (in.rec) return in.rec[k].w ? in.second[in.rec[k].y] : INT32_MIN;
    return in.second[a];
}

// the largest r < n_contigs with contig_begin[r] <= x (upper_bound - 1; contig_begin[0] = 0)
__host__ __device__ __forceinline__ uint32_t contig_of(const uint32_t* __restrict__ cb, uint32_t n_contigs, uint32_t x)
{
    uint32_t lo = 0u, hi = n_contigs;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cb[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

enum { BAM_UNALIGNED = 0, BAM_MAPPED = 1, BAM_OFF_CONTIG = 2, BAM_UNFINISHED = 3 };

struct BamPlace {
    uint32_t state;                                 // BAM_*
    int32_t  ref, pos;                              // mapped only
    uint32_t rlen;                                  // M + D
    uint32_t strand;
};

// the placement rule of nvb_bam_records for alignment a
__host__ __device__ inline BamPlace bam_place(const BamIn& in, uint32_t a)
{
    BamPlace p; p.state = BAM_UNALIGNED; p.ref = -1; p.pos = -1; p.rlen = 0u; p.strand = 0u;
    if (in.n_ops[a] == 0u) return p;
    const uint32_t nc = in.n_cigar[a];
    if (in.edits[4u * (size_t)a] == FINISH_BAD || nc > in.max_cigar || nc > 65535u || in.md_len[a] > in.max_md) { p.state = BAM_UNFINISHED; return p; }
    const uint32_t* cg = in.cigar + (size_t)a * in.max_cigar;
    uint32_t rlen = 0u;
    for (uint32_t k = 0; k < nc; ++k) {
        const uint32_t c = cg[k], op = c & 15u;
        if (op == 0u || op == 2u) rlen += c >> 4;
    }
    const uint32_t bx = in.begin[a].x;
    const uint32_t r = contig_of(in.contig_begin, in.n_contigs, bx);
    const uint32_t cend = in.contig_begin[r + 1u];
    if (bx >= cend || (uint64_t)bx + rlen > cend) { p.state = BAM_OFF_CONTIG; return p; }
    p.state = BAM_MAPPED; p.ref = (int32_t)r; p.pos = (int32_t)(bx - in.contig_begin[r]); p.rlen = rlen; p.strand = in.strand[a] ? 1u : 0u;
    return p;
}

__host__ __device__ __forceinline__ uint32_t bam_name_len(const BamIn& in, uint32_t j)
{
    const uint32_t l = in.name_off[j + 1u] - in.name_off[j];
    return l < BAM_MAX_NAME ? l : BAM_MAX_NAME;
}

// tag bytes of mapped alignment a with second score xs (bam_xs): NM, AS, [XS], XM, XO, XG as integer tags; MD:Z (when not empty) and,
// in nvb_bam_records_all, NH follow them
__host__ __device__ __forceinline__ uint32_t bam_int_tags_bytes(const BamIn& in, uint32_t a, int32_t xs)
{
    const uint32_t* e = in.edits + 4u * (size_t)a;
    uint32_t b = 15u + tag_int_bytes(e[0]) + tag_int_bytes(in.score[a]) + tag_int_bytes(e[1]) + tag_int_bytes(e[2]) + tag_int_bytes(e[3]);
    if (xs != INT32_MIN) b += 3u + tag_int_bytes(xs);
    return b;
}

// the 32-byte core of record k (the eight words bam_write1 writes after block_size) and the record's size in bytes, block_size included
__host__ __device__ inline uint64_t bam_plan_record(const BamIn& in, uint32_t k, const BamPlace& me, const BamPlace* mate, uint32_t* w)
{
    const uint32_t a = bam_alignment(in, k);
    const bool mapped = me.state == BAM_MAPPED;
    uint32_t flag = mapped ? (me.strand ? 0x10u : 0u) : 0x4u;
    int32_t ref = -1, pos = -1, nref = -1, npos = -1, tlen = 0;
    uint32_t bin = 4680u;
    if (mate) {
        const bool mm = mate->state == BAM_MAPPED;
        flag |= 0x1u | ((k & 1u) ? 0x80u : 0x40u);
        const uint32_t pf = in.pair_flags[k >> 1];
        if ((pf == NVB_PAIR_CONCORDANT || pf == NVB_PAIR_RESCUED_MATE1 || pf == NVB_PAIR_RESCUED_MATE2) && mapped && mm) flag |= 0x2u;
        if (!mm) flag |= 0x8u;
        else if (mate->strand) flag |= 0x20u;
        if (mapped) {
            ref = me.ref; pos = me.pos;
            if (mm) {
                nref = mate->ref; npos = mate->pos;
                if (mate->ref == me.ref) {
                    const int64_t e0 = (int64_t)me.pos + me.rlen, e1 = (int64_t)mate->pos + mate->rlen;
                    const int64_t lo = me.pos < mate->pos ? me.pos : mate->pos;
                    const int32_t t = (int32_t)((e0 > e1 ? e0 : e1) - lo);
                    tlen = (me.pos < mate->pos || (me.pos == mate->pos && !(k & 1u))) ? t : -t;
                }
            } else {
                nref = me.ref; npos = me.pos;
            }
        } else if (mm) {
            ref = nref = mate->ref; pos = npos = mate->pos;
            bin = bam_reg2bin(pos, (int64_t)pos + 1);
        }
    } else if (mapped) {
        ref = me.ref; pos = me.pos;
    }
    const uint32_t nc = mapped ? in.n_cigar[a] : 0u;
    if (mapped) bin = bam_reg2bin(pos, (int64_t)pos + me.rlen);
    uint32_t mapq = mapped ? (in.mapq ? in.mapq[a] : 255u) : 0u;
    if (in.rec && mapped) {                         // nvb_bam_records_all: the read's MAPQ on its primary record, 255 and 0x100 on the others
        mapq = in.rec[k].w && in.mapq ? in.mapq[in.rec[k].y] : 255u;
        if (!in.rec[k].w) flag |= 0x100u;
    }
    const uint32_t l_name = bam_name_len(in, bam_name(in, k)) + 1u;
    const uint32_t l_seq = str_len(in.reads, bam_seq(in, k));
    w[0] = (uint32_t)ref; w[1] = (uint32_t)pos;
    w[2] = bin << 16 | mapq << 8 | l_name;
    w[3] = flag << 16 | nc;
    w[4] = l_seq;
    w[5] = (uint32_t)nref; w[6] = (uint32_t)npos; w[7] = (uint32_t)tlen;
    uint64_t size = BAM_FIXED + l_name + 4u * nc + ((l_seq + 1u) >> 1) + l_seq;
    if (mapped) {
        size += bam_int_tags_bytes(in, a, bam_xs(in, k, a));
        if (in.md_len[a]) size += 4u + in.md_len[a];
        if (in.rec) size += 3u + tag_int_bytes(in.rec[k].z);
    }
    return size;
}

// plan unit u: read u (single end) or pair u (both mates, records 2u and 2u + 1).  Writes the cores (8 words per record) and sizes of
// its records; adds (mapped, off-contig, unfinished) of them to cnt.
__host__ __device__ inline void bam_plan_unit(const BamIn& in, uint32_t u, uint32_t* __restrict__ cores, uint64_t* __restrict__ sizes, uint32_t cnt[3])
{
    if (!in.pair_flags) {
        const BamPlace p = bam_place(in, u);
        sizes[u] = bam_plan_record(in, u, p, nullptr, cores + 8u * (size_t)u);
        cnt[0] += p.state == BAM_MAPPED; cnt[1] += p.state == BAM_OFF_CONTIG; cnt[2] += p.state == BAM_UNFINISHED;
        return;
    }
    const BamPlace p0 = bam_place(in, u), p1 = bam_place(in, (in.n >> 1) + u);
    sizes[2u * u]      = bam_plan_record(in, 2u * u, p0, &p1, cores + 16u * (size_t)u);
    sizes[2u * u + 1u] = bam_plan_record(in, 2u * u + 1u, p1, &p0, cores + 16u * (size_t)u + 8u);
    cnt[0] += (p0.state == BAM_MAPPED) + (p1.state == BAM_MAPPED);
    cnt[1] += (p0.state == BAM_OFF_CONTIG) + (p1.state == BAM_OFF_CONTIG);
    cnt[2] += (p0.state == BAM_UNFINISHED) + (p1.state == BAM_UNFINISHED);
}

// nvb_bam_records_all, read r (alignments [first[r], first[r + 1]), stored when first[r + 1] <= capacity): its mapped alignments in rank
// order, or one unmapped record.  rec_first == NULL: only count -- returns the records, adds (mapped, off-contig, unfinished or beyond the
// capacity) to cnt.  Else writes records rec_first[r] .. : rec (as BamIn.rec, which must point at it), cores and sizes
__host__ __device__ inline uint32_t bam_plan_read_all(const BamIn& in, uint32_t r, const uint32_t* first, uint32_t capacity, const uint32_t* rec_first,
                                                      uint4* rec, uint32_t* __restrict__ cores, uint64_t* __restrict__ sizes, uint32_t cnt[3])
{
    const uint32_t b = first[r], e = first[r + 1];
    const bool stored = e <= capacity;
    uint32_t m = 0;
    if (stored)
        for (uint32_t a = b; a < e; ++a) {
            const uint32_t st = bam_place(in, a).state;
            m += st == BAM_MAPPED;
            if (!rec_first) { cnt[1] += st == BAM_OFF_CONTIG; cnt[2] += st == BAM_UNFINISHED; }
        }
    if (!rec_first) { cnt[0] += m; cnt[2] += !stored; return m ? m : 1u; }
    uint32_t k = rec_first[r];
    if (!m) {
        BamPlace p; p.state = BAM_UNALIGNED; p.ref = -1; p.pos = -1; p.rlen = 0u; p.strand = 0u;
        rec[k] = make_uint4(BAM_NO_ALN, r, 0u, 1u);
        sizes[k] = bam_plan_record(in, k, p, nullptr, cores + 8u * (size_t)k);
        return 1u;
    }
    for (uint32_t a = b; a < e; ++a) {
        const BamPlace p = bam_place(in, a);
        if (p.state != BAM_MAPPED) continue;
        rec[k] = make_uint4(a, r, m, k == rec_first[r] ? 1u : 0u);
        sizes[k] = bam_plan_record(in, k, p, nullptr, cores + 8u * (size_t)k);
        ++k;
    }
    return m;
}

__host__ __device__ __forceinline__ void put32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
__host__ __device__ __forceinline__ uint32_t nt16(uint32_t code, uint32_t is_n) { return is_n ? 15u : 1u << code; }
// one integer tag (name c0 c1, htslib's type for v, little-endian value); returns the byte after it
__host__ __device__ __forceinline__ uint8_t* put_int_tag(uint8_t* t, char c0, char c1, int64_t v)
{
    const uint32_t nb = tag_int_bytes(v);
    t[0] = (uint8_t)c0; t[1] = (uint8_t)c1; t[2] = (uint8_t)tag_int_type(v, nb);
    for (uint32_t b = 0; b < nb; ++b) t[3u + b] = (uint8_t)((uint64_t)v >> (8u * b));
    return t + 3u + nb;
}

// Compose record k (core w, size bytes) at dst.  The work is split over nl lanes, lane `lane` writing its share; every byte is written by
// exactly one lane, so lanes 0 .. nl - 1 run one after another (the host) give what a warp gives.  SEQ: CHUNK symbols per lane step
// from the packed read (read_chunk), mirrored and complemented for strand 1 as finish_alignment does.
template <int BITS, bool BE>
__host__ __device__ __forceinline__ void bam_compose(const BamIn& in, uint32_t k, const uint32_t* __restrict__ w, uint32_t size, uint8_t* __restrict__ dst,
                                            uint32_t lane, uint32_t nl)
{
    constexpr uint32_t CHUNK = ReadChunk<BITS, BE>::CHUNK;
    const uint32_t a = bam_alignment(in, k);
    for (uint32_t i = lane; i < 9u; i += nl) put32(dst + 4u * i, i ? w[i - 1u] : size - 4u);
    const uint32_t l_name = w[2] & 0xFFu, flag = w[3] >> 16, nc = w[3] & 0xFFFFu, l = w[4];
    const bool mapped = !(flag & 0x4u);
    const uint32_t strand = (flag >> 4) & 1u;
    uint8_t* p = dst + BAM_FIXED;
    const char* name = in.names + in.name_off[bam_name(in, k)];
    for (uint32_t i = lane; i < l_name; i += nl) p[i] = i + 1u < l_name ? (uint8_t)name[i] : 0u;
    p += l_name;
    const uint32_t* cg = in.cigar + (size_t)a * in.max_cigar;
    for (uint32_t i = lane; i < nc; i += nl) put32(p + 4u * i, cg[i]);
    p += 4u * nc;
    const uint32_t off = str_off(in.reads, bam_seq(in, k));
    for (uint32_t y = lane * CHUNK; y < l; y += nl * CHUNK) {
        const uint32_t cnt = l - y < CHUNK ? l - y : CHUNK;
        uint32_t codes, nflags;
        if (strand == 0u) {
            read_chunk<BITS, BE>(in.reads.words, off + y, cnt, codes, nflags);
        } else {
            read_chunk<BITS, BE>(in.reads.words, off + (l - y - cnt), cnt, codes, nflags);
            codes  = ~reverse_2bit_groups(codes) >> (32u - 2u * cnt);
            nflags = reverse_2bit_groups(nflags) >> (32u - 2u * cnt);
        }
        for (uint32_t j = 0; j < cnt; j += 2u) {
            const uint32_t s0 = 2u * (cnt - 1u - j);
            uint32_t b = nt16((codes >> s0) & 3u, (nflags >> s0) & 1u) << 4;
            if (j + 1u < cnt) b |= nt16((codes >> (s0 - 2u)) & 3u, (nflags >> (s0 - 2u)) & 1u);
            p[(y + j) >> 1] = (uint8_t)b;
        }
    }
    p += (l + 1u) >> 1;
    for (uint32_t i = lane; i < l; i += nl) p[i] = in.quals ? in.quals[off + (strand ? l - 1u - i : i)] : 0xFFu;
    p += l;
    if (!mapped) return;
    const uint32_t* e = in.edits + 4u * (size_t)a;
    const int32_t xs = bam_xs(in, k, a);
    if (lane == 0u) {
        uint8_t* t = put_int_tag(p, 'N', 'M', e[0]);
        t = put_int_tag(t, 'A', 'S', in.score[a]);
        if (xs != INT32_MIN) t = put_int_tag(t, 'X', 'S', xs);
        t = put_int_tag(t, 'X', 'M', e[1]);
        t = put_int_tag(t, 'X', 'O', e[2]);
        put_int_tag(t, 'X', 'G', e[3]);
    }
    const uint32_t ml = in.md_len[a];
    p += bam_int_tags_bytes(in, a, xs);
    if (ml) {
        const char* md = in.md + (size_t)a * in.max_md;
        if (lane == 0u) { p[0] = 'M'; p[1] = 'D'; p[2] = 'Z'; p[3u + ml] = 0u; }
        for (uint32_t i = lane; i < ml; i += nl) p[3u + i] = (uint8_t)md[i];
        p += 4u + ml;
    }
    if (in.rec && lane == 0u) put_int_tag(p, 'N', 'H', in.rec[k].z);
}

} // namespace nvb
