// finish_core.cuh -- per-alignment routine of nvb_finish_alignments (finish.cu) that the tests also run on the host
// (tests/host/finish_harness.cu): a traced alignment (ops END -> START, begin, strand) and the read and genome beside it become a BAM
// CIGAR with soft clips, the SAM MD:Z value and the edit counts NM / XM / XO / XG.
#pragma once
#include "pipeline_core.cuh"

namespace nvb {

constexpr uint32_t FINISH_BAD = 0xFFFFFFFFu;        // edits[0] of an alignment that cannot be finished

__host__ __device__ __forceinline__ uint32_t nvb_brev(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __brev(x);
#else
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4);
    x = ((x >> 8) & 0x00FF00FFu) | ((x & 0x00FF00FFu) << 8);
    return (x >> 16) | (x << 16);
#endif
}
// the 16 two-bit groups of x in reverse order (the bits inside each group keep their order)
__host__ __device__ __forceinline__ uint32_t reverse_2bit_groups(uint32_t x)
{
    const uint32_t y = nvb_brev(x);
    return ((y >> 1) & 0x55555555u) | ((y & 0x55555555u) << 1);
}
// even bits of the low 2 * cnt bits (one flag per symbol of a cnt-symbol chunk), cnt in [0, 16]
__host__ __device__ __forceinline__ uint32_t chunk_flags(uint32_t cnt) { return cnt >= 16u ? 0x55555555u : ((1u << (2u * cnt)) - 1u) & 0x55555555u; }

// Symbols [a, a + cnt) of a packed read stream, cnt <= CHUNK: their 2-bit codes in the low 2 * cnt bits, symbol a highest, and a flag
// at bit 2 * (cnt - 1 - k) for every symbol a + k that is an N (> 3).  2-bit big-endian reads are one funnel shift; 4-bit big-endian
// reads are one funnel shift of 8 nibbles; other layouts are gathered symbol by symbol.
template <int BITS, bool BE> struct ReadChunk { static constexpr uint32_t CHUNK = (BITS == 4 && BE) ? 8u : 16u; };

template <int BITS, bool BE>
__host__ __device__ __forceinline__ void read_chunk(const uint32_t* __restrict__ words, uint32_t a, uint32_t cnt, uint32_t& codes, uint32_t& nflags)
{
    if (BITS == 2 && BE) {
        codes = be2_window(words, a, cnt) >> (32u - 2u * cnt); nflags = 0u;
    } else if (BITS == 4 && BE) {
        const uint32_t wi = a >> 3, r = a & 7u, sh = 4u * r;
        const uint32_t w0 = words[wi], w1 = (r + cnt > 8u) ? words[wi + 1u] : 0u;
        const uint32_t x = r ? ((w0 << sh) | (w1 >> (32u - sh))) : w0;            // 8 nibbles, symbol a on top
        codes  = squeeze_nibbles(x) >> (16u - 2u * cnt);
        nflags = squeeze_nibbles(((x >> 2) | (x >> 3)) & 0x11111111u) >> (16u - 2u * cnt);
    } else {
        codes = 0u; nflags = 0u;
#pragma unroll 1
        for (uint32_t k = 0; k < cnt; ++k) {
            const uint32_t c = sym_at<BITS, BE>(words, a + k);
            codes = (codes << 2) | (c & 3u); nflags = (nflags << 2) | (c > 3u ? 1u : 0u);
        }
    }
}

// Bounded writers of one alignment's outputs: everything is counted, only what fits is stored.
struct FinishOut {
    uint32_t* cigar; uint32_t max_cigar, n_cigar;
    char*     md;    uint32_t max_md, md_len;
    __host__ __device__ __forceinline__ void run(uint32_t len, uint32_t op) {
        if (n_cigar < max_cigar) cigar[n_cigar] = (len << 4) | op;
        ++n_cigar;
    }
    __host__ __device__ __forceinline__ void chr(uint32_t c) {
        if (md_len < max_md) md[md_len] = (char)c;
        ++md_len;
    }
    __host__ __device__ __forceinline__ void num(uint32_t v) {           // decimal, no leading zeros ("0" for 0)
        uint32_t p = 1u;
        while (v / p >= 10u) p *= 10u;
        for (; p; p /= 10u) chr('0' + (v / p) % 10u);
    }
};

__host__ __device__ __forceinline__ uint32_t base_char(uint32_t c) { return (0x54474341u >> (8u * c)) & 0xFFu; }   // "ACGT"[c]

// Finish one traced alignment.  read = symbols [off, off + len) of the caller's read stream; strand != 0: the alignment is of its reverse
// complement (symbol p = c < 4 ? 3 - c : c of caller symbol len - 1 - p); ops[0, n_ops) END -> START (0 M, 1 I, 2 D); begin (bx, by) =
// (genome coordinate of the first aligned genome symbol, first aligned read symbol of the strand's string); genome = 2-bit big-endian,
// genome_len symbols.  Writes the BAM CIGAR (len << 4 | op: 0 M, 1 I, 2 D, 4 S, START -> END) and the MD:Z value (bounded by max_cigar /
// max_md, the full counts in n_cigar / md_len) and edits[0..3] = NM, XM, XO, XG.  An M column at a genome coordinate >= genome_len is a
// mismatch against N.  Not finishable (n_ops > max_ops, bx == 0xFFFFFFFF, an op byte > 2, more read symbols consumed than len - by):
// no CIGAR, no MD, edits = (0xFFFFFFFF, 0, 0, 0).  Reads only ops[0, min(n_ops, max_ops)), the read's own symbols and genome symbols
// below genome_len.
template <int BITS, bool BE>
__host__ __device__ inline void finish_alignment(const uint32_t* __restrict__ genome, const uint32_t genome_len,
                                                 const uint32_t* __restrict__ read_words, const uint32_t off, const uint32_t len, const uint32_t strand,
                                                 const uint8_t* __restrict__ ops, const uint32_t n_ops, const uint32_t max_ops,
                                                 const uint32_t bx, const uint32_t by, FinishOut& o, uint32_t* __restrict__ edits)
{
    constexpr uint32_t CHUNK = ReadChunk<BITS, BE>::CHUNK;
    o.n_cigar = 0u; o.md_len = 0u;
    uint32_t nm = 0u, xm = 0u, xo = 0u, xg = 0u;
    if (n_ops == 0u) { edits[0] = edits[1] = edits[2] = edits[3] = 0u; return; }
    // pass 1: the column counts, and whether the alignment can be finished at all
    bool bad = n_ops > max_ops || bx == 0xFFFFFFFFu || by > len;
    uint32_t n_m = 0u, n_i = 0u, n_d = 0u;
    for (uint32_t i = 0; i < n_ops && !bad; ++i) {
        const uint32_t op = ops[i];
        n_m += op == 0u; n_i += op == 1u; n_d += op == 2u; bad |= op > 2u;
    }
    if (bad || n_m + n_i > len - by) { edits[0] = FINISH_BAD; edits[1] = edits[2] = edits[3] = 0u; return; }

    // pass 2: the runs START -> END
    if (by) o.run(by, 4u);
    uint32_t x = bx, y = by, mrun = 0u;                      // genome / read position, matches since the last MD token
    for (uint32_t i = n_ops; i > 0u;) {
        const uint32_t op = ops[i - 1u];
        uint32_t k = 1u;
        while (k < i && ops[i - 1u - k] == op) ++k;
        i -= k;
        o.run(k, op);
        if (op == 1u) { y += k; nm += k; ++xo; xg += k - 1u; continue; }
        if (op == 2u) {
            o.num(mrun); mrun = 0u; o.chr('^');
            for (uint32_t c = 0; c < k; ++c, ++x) o.chr(x < genome_len ? base_char(sym_at<2, true>(genome, x)) : 'N');
            nm += k; ++xo; xg += k - 1u;
            continue;
        }
        // M run of k columns: CHUNK columns per step, read (reverse-complemented on the fly) XOR genome, mismatches by clz
        for (uint32_t c0 = 0; c0 < k; c0 += CHUNK) {
            const uint32_t cnt = k - c0 < CHUNK ? k - c0 : CHUNK;
            uint32_t codes, nflags;
            if (strand == 0u) {
                read_chunk<BITS, BE>(read_words, off + y, cnt, codes, nflags);
            } else {
                read_chunk<BITS, BE>(read_words, off + (len - y - cnt), cnt, codes, nflags);
                codes  = ~reverse_2bit_groups(codes) >> (32u - 2u * cnt);
                nflags = reverse_2bit_groups(nflags) >> (32u - 2u * cnt);
            }
            const uint32_t cg = x < genome_len ? (genome_len - x < cnt ? genome_len - x : cnt) : 0u;   // columns inside the genome
            const uint32_t g = cg ? be2_window(genome, x, cg) >> (32u - 2u * cnt) : 0u;
            const uint32_t dx = codes ^ g;
            // one flag per mismatched column: a differing symbol, a read N, or a column past the genome's end (a mismatch against N)
            uint32_t d = ((dx | (dx >> 1)) & chunk_flags(cnt)) | nflags | chunk_flags(cnt - cg);
            uint32_t prev = 0u;                              // first column of the chunk not yet counted
            while (d) {
                const uint32_t bit = 31u - nvb_clz(d);       // the flags sit on even bits
                d ^= 1u << bit;
                const uint32_t p = cnt - 1u - (bit >> 1);    // column of the chunk
                mrun += p - prev; prev = p + 1u;
                o.num(mrun); mrun = 0u;
                o.chr(p < cg ? base_char((g >> bit) & 3u) : 'N');
                ++xm;
            }
            mrun += cnt - prev;
            x += cnt; y += cnt;
        }
    }
    o.num(mrun);
    if (len - y) o.run(len - y, 4u);
    edits[0] = xm + nm; edits[1] = xm; edits[2] = xo; edits[3] = xg;
}

} // namespace nvb
