// pipeline_core.cuh -- per-thread routines of the seed + extend composition that tests also run on the host
// (tests/host/host_harness.cu, tests/host/mapq_harness.cu), like fm_core.cuh / gotoh_core.cuh.
#pragma once
#include "fm_core.cuh"

namespace nvb {

__host__ __device__ __forceinline__ uint32_t nvb_clz(uint32_t x) {        // x != 0
#ifdef __CUDA_ARCH__
    return (uint32_t)__clz((int)x);
#else
    return (uint32_t)__builtin_clz(x);
#endif
}

// one bit per differing symbol (bit 2k = symbol cnt-1-k) of read[i, i+cnt) against text[t+i, ...); both 2-bit big-endian streams
__host__ __device__ __forceinline__ uint32_t job_diff_bits(const uint32_t* __restrict__ str_words, const uint32_t* __restrict__ genome,
                                                           const uint32_t po, const uint32_t t, const uint32_t i, const uint32_t cnt)
{
    const uint32_t x = (be2_window(str_words, po + i, cnt) ^ be2_window(genome, t + i, cnt)) >> (32u - 2u * cnt);
    return (x | (x >> 1)) & 0x55555555u;
}
// number of differing symbols on the diagonal starting at text position t; counting stops once it exceeds `limit`
__host__ __device__ __forceinline__ uint32_t job_differences(const uint32_t* __restrict__ str_words, const uint32_t* __restrict__ genome,
                                                             const uint32_t po, const uint32_t M, const uint32_t t, const uint32_t limit)
{
    uint32_t mm = 0;
    for (uint32_t i = 0; i < M && mm <= limit; i += 16u) mm += nvb_popc(job_diff_bits(str_words, genome, po, t, i, M - i < 16u ? M - i : 16u));
    return mm;
}

// the bits of rows [lo, hi] in a job_diff_bits word that holds rows [w0, w0 + cnt) (row w0 + cnt - 1 - k at bit 2k); 0 when none
__host__ __device__ __forceinline__ uint32_t diff_row_mask(const uint32_t w0, const uint32_t cnt, const uint32_t lo, const uint32_t hi)
{
    const uint32_t a = lo > w0 ? lo : w0, b = hi < w0 + cnt - 1u ? hi : w0 + cnt - 1u;
    if (a > b) return 0u;
    return ((2u << (2u * (w0 + cnt - 1u - a))) - 1u) & ~((1u << (2u * (w0 + cnt - 1u - b))) - 1u);
}
// first and last differing row in [lo, hi] on the diagonal starting at text position t (hi + 1 and lo - 1 when there is none)
__host__ __device__ inline void job_diff_span(const uint32_t* __restrict__ str_words, const uint32_t* __restrict__ genome, const uint32_t po,
                                              const uint32_t t, const uint32_t lo, const uint32_t hi, int32_t& first, int32_t& last)
{
    first = (int32_t)hi + 1; last = (int32_t)lo - 1;
    for (uint32_t i = lo; i <= hi; i += 16u) {
        const uint32_t cnt = hi + 1u - i < 16u ? hi + 1u - i : 16u;
        const uint32_t d = job_diff_bits(str_words, genome, po, t, i, cnt);
        if (!d) continue;
        if (first > (int32_t)hi) first = (int32_t)(i + cnt - 1u - ((31u - nvb_clz(d)) >> 1));
        last = (int32_t)(i + cnt - 1u - ((31u - nvb_clz(d & (0u - d))) >> 1));
    }
}
// the 16 symbols at symbol offset off (< 48) of the four consecutive text words g0..g3
__host__ __device__ __forceinline__ uint32_t text_window16(const uint32_t g0, const uint32_t g1, const uint32_t g2, const uint32_t g3, const uint32_t off)
{
    const uint32_t idx = off >> 4, sh = 2u * (off & 15u);
    const uint32_t hi = idx == 0u ? g0 : (idx == 1u ? g1 : g2), lo = idx == 0u ? g1 : (idx == 1u ? g2 : g3);
    return sh ? ((hi << sh) | (lo >> (32u - sh))) : hi;
}

constexpr uint32_t SHORTCUT_WORDS = 10;     // read words per load batch of gapless_job_shortcut's diagonal pass (a 150 bp read: one batch)

// Exact shortcut of the LOCAL banded extension for a read that lies on its seed's diagonal with few differences -- most reads of a real
// run.  With m = match > 0 > s = mismatch, gap-open penalties < 0 and gap-extension penalties <= 0, every gap costs at least
// o = -max(pattern_gap_open, text_gap_open) > 0.  Let T be the best segment of the seed's diagonal j0 and delta = m * M - T:
//   * an alignment without a gap lies on ONE band diagonal, and the best of those is the maximum-sum segment of that diagonal's
//     match / mismatch scores (H along the diagonal with only the diagonal move: h = max(0, h + s)); another diagonal reaches T only
//     with at most delta / m differences;
//   * an alignment with g >= 1 gaps, q mismatched columns and u read rows outside its aligned columns (clipped, or inside an
//     insertion) scores at most  m * M - m * u - (m - s) * q - g * o,  so it reaches T only if  m * u + (m - s) * q + g * o <= delta.
// delta < o: no gapped alignment reaches T.  o <= delta < min(2 o, o + m - s) (the one-gap check, on unless one_gap = false): one that
// does has exactly one gap, no mismatch and u <= U = (delta - o) / m -- two exact pieces on band diagonals d1 != d2, the first starting
// at a row <= U, the second ending at a row >= M - 1 - U, at most U rows between them.  With F_d / B_d the first / last differing row of
// diagonal d in [U, M - 1 - U] (M - U / U - 1 when none), the first piece ends before F_d1 and the second starts after B_d2, so such an
// alignment needs  B_d2 - F_d1 <= U - 1.  When no band diagonal and no such pair can reach T, T is the band's maximum and every cell
// holding it lies on j0: the DP's result is (T, last row where h == T) -- BestSink keeps the last maximal cell in row-major order
// (sink_inl.h:39-65).  A read without any difference (score m * M, only reachable in the last row) may tie with other equal diagonals
// (tandem repeats): the largest one wins.
// The job: read = 2-bit big-endian symbols [po, po + M) of str_words (po a multiple of 16), window = text[to, to + N), the seed's
// diagonal band/2 into the window (pipe_resolve_reads_kernel cuts it there; a window clamped at the text start, to == 0, has it somewhere
// below and is left to the DP), band <= 32.  Returns true and (score, sink = (text end, pattern end), both 1-based ends as BestSink
// reports them) when the result is proven; false = run the DP.  Only full windows qualify (N >= M + band - 1: no pad symbol in the band).
__host__ __device__ inline bool gapless_job_shortcut(const uint32_t* __restrict__ str_words, const uint32_t* __restrict__ genome,
                                                     const uint32_t po, const uint32_t M, const uint32_t to, const uint32_t N, const uint32_t band,
                                                     const int32_t match, const int32_t mismatch, const int32_t max_gap_open,
                                                     int32_t& score, uint32_t& sink_x, uint32_t& sink_y, const bool one_gap = true)
{
    if (M < 1u || to == 0u || N < M + band - 1u) return false;
    const uint32_t j0 = band / 2u;
    const int32_t o = -max_gap_open, lim = !one_gap ? o : (o + match - mismatch < 2 * o ? o + match - mismatch : 2 * o);   // claimed: delta < lim
    // differences the seed's diagonal may have and still be claimed: each one adds at least match to delta
    const uint32_t mm_max = (uint32_t)((lim - 1) / match);
    // one pass over the seed's diagonal: its differences (at most mm_max, else the DP), its first two and last two differing rows, and,
    // from the runs of equal symbols between them, the maximum-sum segment with the LAST end among equals.  (mismatch < 0, so h peaks at
    // the ends of runs; a symbol-by-symbol version of this loop cost 1,500 warp instructions per job)
    // The read and diagonal words are loaded SHORTCUT_WORDS (+1) at a time, every load of a batch issued before the first comparison, so
    // a job pays one memory round trip per batch instead of one per 16 symbols (job_diff_bits on the same words: the read starts on a
    // word, the diagonal is a funnel shift of two consecutive text words, and no word past the window's last one is touched).
    int32_t h = 0, best = 0, f1 = (int32_t)M, f2 = (int32_t)M, l1 = -1, l2 = -1; uint32_t end = 0, prev = 0, mm0 = 0;
    const uint32_t wr = po >> 4, wt = (to + j0) >> 4, sht = 2u * ((to + j0) & 15u), wlast = (to + N - 1u) >> 4;
    for (uint32_t kb = 0; kb * 16u < M && mm0 <= mm_max; kb += SHORTCUT_WORDS) {
        uint32_t rw[SHORTCUT_WORDS], tw[SHORTCUT_WORDS + 1];
#pragma unroll
        for (uint32_t q = 0; q < SHORTCUT_WORDS; ++q) rw[q] = (kb + q) * 16u < M ? str_words[wr + kb + q] : 0u;
#pragma unroll
        for (uint32_t q = 0; q <= SHORTCUT_WORDS; ++q) tw[q] = wt + kb + q <= wlast ? genome[wt + kb + q] : 0u;
#pragma unroll
        for (uint32_t q = 0; q < SHORTCUT_WORDS; ++q) {
            const uint32_t i = (kb + q) * 16u;
            if (i >= M || mm0 > mm_max) break;
            const uint32_t cnt = M - i < 16u ? M - i : 16u;
            const uint32_t x = (rw[q] ^ (sht ? (tw[q] << sht) | (tw[q + 1] >> (32u - sht)) : tw[q])) >> (32u - 2u * cnt);
            uint32_t d = (x | (x >> 1)) & 0x55555555u;
            while (d && mm0 <= mm_max) {
                const uint32_t bit = 31u - nvb_clz(d);                      // highest set bit = first differing symbol of the word
                const uint32_t p = i + (cnt - 1u - (bit >> 1));
                d &= ~(1u << bit);
                h += match * (int32_t)(p - prev);
                if (h >= best) { best = h; end = p; }
                h += mismatch; h = h > 0 ? h : 0;
                if (mm0 == 0u) f1 = (int32_t)p; else if (mm0 == 1u) f2 = (int32_t)p;
                l2 = l1; l1 = (int32_t)p;
                prev = p + 1u; ++mm0;
            }
        }
    }
    if (mm0 > mm_max) return false;
    h += match * (int32_t)(M - prev);
    if (h >= best) { best = h; end = M; }
    const int32_t delta = match * (int32_t)M - best;
    if (delta >= lim) return false;
    // One-gap check (delta >= o): F and B of every band diagonal, keeping the two largest F and the two smallest B.  For j0 they come from
    // its first two / last two differences (a third one inside the clip rows makes F larger or B smaller than it is: the check only
    // claims less); for the others from the first and the last 16 read symbols against four text words each, with a full comparison
    // only for a diagonal without a difference there (j0's neighbours in a tandem repeat).
    const bool gap1 = delta >= o;
    const uint32_t U = gap1 ? (uint32_t)((delta - o) / match) : 0u;
    if (gap1 && 2u * U + 1u > M) return false;                              // [U, M - 1 - U] is empty: every pair qualifies
    const uint32_t hi = M - 1u - U;
    int32_t fa = f1 >= (int32_t)U ? f1 : (f2 >= (int32_t)U ? f2 : (int32_t)(M - U)), ba = l1 <= (int32_t)hi ? l1 : (l2 <= (int32_t)hi ? l2 : (int32_t)U - 1);
    fa = fa > (int32_t)hi ? (int32_t)(M - U) : fa; ba = ba < (int32_t)U ? (int32_t)U - 1 : ba;
    int32_t fb = INT_MIN, bb = INT_MAX; uint32_t fd = j0, bd = j0;          // (largest F, its diagonal, second largest; the same for B)
    // Can another band diagonal reach `best`?  Only with at most t differences (match * equal positions bounds its score).  The first 16
    // symbols decide that for nearly every diagonal: they are compared against all band offsets from four text words held in registers
    // (a full comparison only follows for a diagonal they do not rule out).
    const bool perfect = (mm0 == 0u);
    const uint32_t t = (uint32_t)(delta / match);
    const uint32_t c16 = M < 16u ? M : 16u;
    const uint32_t r0 = be2_window(str_words, po, c16) >> (32u - 2u * c16);
    const uint32_t wi = to >> 4, r = to & 15u, wl = (to + N - 1u) >> 4;      // wl: last word holding a window symbol
    const uint32_t g0 = genome[wi], g1 = (wi + 1u <= wl) ? genome[wi + 1u] : 0u;
    const uint32_t g2 = (wi + 2u <= wl) ? genome[wi + 2u] : 0u, g3 = (wi + 3u <= wl) ? genome[wi + 3u] : 0u;
    // the last c16 read symbols and the text words their band offsets lie in
    uint32_t rE = 0, e0 = 0, e1 = 0, e2 = 0, e3 = 0, mF = 0, mB = 0;
    const uint32_t te = to + M - c16, we = te >> 4;
    if (gap1) {
        rE = be2_window(str_words, po + M - c16, c16) >> (32u - 2u * c16);
        e0 = genome[we]; e1 = (we + 1u <= wl) ? genome[we + 1u] : 0u; e2 = (we + 2u <= wl) ? genome[we + 2u] : 0u; e3 = (we + 3u <= wl) ? genome[we + 3u] : 0u;
        mF = diff_row_mask(0u, c16, U, hi); mB = diff_row_mask(M - c16, c16, U, hi);
    }
    uint32_t jtop = j0;                                                     // largest diagonal without a difference
    for (uint32_t jj = 0; jj < band; ++jj) {                                // band <= 32: offsets < 48
        if (jj == j0) continue;
        const uint32_t x = (text_window16(g0, g1, g2, g3, r + jj) >> (32u - 2u * c16)) ^ r0, dx = (x | (x >> 1)) & 0x55555555u;
        if (gap1) {
            const uint32_t y = (text_window16(e0, e1, e2, e3, (te & 15u) + jj) >> (32u - 2u * c16)) ^ rE, dy = (y | (y >> 1)) & 0x55555555u & mB;
            int32_t F, B;
            if ((dx & mF) && dy) { F = (int32_t)(c16 - 1u - ((31u - nvb_clz(dx & mF)) >> 1)); B = (int32_t)(M - 1u - ((31u - nvb_clz(dy & (0u - dy))) >> 1)); }
            else job_diff_span(str_words, genome, po, to + jj, U, hi, F, B);
            if (F > fa) { fb = fa; fa = F; fd = jj; } else if (F > fb) fb = F;
            if (B < ba) { bb = ba; ba = B; bd = jj; } else if (B < bb) bb = B;
        }
        if (nvb_popc(dx) > t) continue;
        if (job_differences(str_words, genome, po, M, to + jj, t) > t) continue;
        if (!perfect) return false;                                         // another diagonal might tie: the DP decides
        if (jj > jtop) jtop = jj;                                           // (another diagonal without a difference)
    }
    // the closest pair d1 != d2: min over them of B_d2 - F_d1
    if (gap1 && (fd != bd ? (int64_t)ba - fa : ((int64_t)ba - fb < (int64_t)bb - fa ? (int64_t)ba - fb : (int64_t)bb - fa)) <= (int64_t)U - 1) return false;
    score = best;
    if (perfect) { sink_x = M + jtop; sink_y = M; }
    else         { sink_x = end + j0; sink_y = end; }
    return true;
}

// Alignment ending at p on strand t is distinct from the best one (bp, bt) of a read of length len: another strand, or an end more than
// len/2 away (nvbio io::distinct_alignments, alignments_inl.h:35-47, in the same unsigned arithmetic)
__host__ __device__ __forceinline__ bool distinct_alignment(uint32_t p, uint32_t t, uint32_t bp, uint32_t bt, uint32_t len)
{
    const uint32_t d = len / 2u;
    return t != bt || p < bp - (bp < d ? bp : d) || p > bp + d;
}

// best-per-read key (64-bit atomicMax; 0 = none): higher score, then smaller tie index -- both paths' tie rule
__host__ __device__ __forceinline__ unsigned long long make_best_key(int32_t score, uint32_t index)
{
    return ((unsigned long long)((uint32_t)score ^ 0x80000000u) << 32) | (unsigned long long)(0xFFFFFFFFu - index);
}
__host__ __device__ __forceinline__ int32_t  best_key_score(unsigned long long key) { return (int32_t)((uint32_t)(key >> 32) ^ 0x80000000u); }
__host__ __device__ __forceinline__ uint32_t best_key_index(unsigned long long key) { return 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull); }

// a scored job is an alignment unless the DP reported it empty (window shorter than the read: NVB_SINK_MIN, sink 0xFFFFFFFF) -- a read
// running more than band/2 symbols past the genome's end gets such a window; it never becomes a best, second-best or pair candidate
__host__ __device__ __forceinline__ bool job_aligned(uint2 sink) { return sink.x != 0xFFFFFFFFu; }

// a scored job that may be reported beside the best alignment: aligned and reaching the read's min score (the candidates of the paired
// MAPQ and of nvb_seed_extend_all)
__host__ __device__ __forceinline__ bool reportable(int32_t score, uint2 sink, int32_t min_score) { return job_aligned(sink) && score >= min_score; }

// nvb_seed_extend_reseed: the first seed of round r starts at r * floor(I / (max_reseed + 1)) (nvBowtie's retry stride,
// mapping_inl.h:553-565)
__host__ __device__ __forceinline__ uint32_t reseed_offset(uint32_t round, uint32_t seed_interval, uint32_t max_reseed)
{
    return round * (seed_interval / (max_reseed + 1u));
}

// nvb_seed_extend_reseed: a read goes on to the next round when its round's seeds found no SA range, their mean range size reached
// rep_seeds (range_sum >= rep_seeds * range_count in wrapping uint32 arithmetic, as map_seeds_kernel and mapping_inl.h:586-588), or its
// best alignment so far does not reach its min score (aligner_init.cu:422-437's mark_unaligned)
__host__ __device__ __forceinline__ bool reseed_read(uint32_t range_sum, uint32_t range_count, uint32_t rep_seeds, bool aligned)
{
    return range_count == 0u || range_sum >= rep_seeds * range_count || !aligned;
}

// (end, strand) of a candidate packed for select_distinct
__host__ __device__ __forceinline__ unsigned long long end_strand(uint32_t end, uint32_t strand) { return ((unsigned long long)end << 1) | (strand & 1u); }

// Selection rule of nvb_seed_extend_all for one read of length len: es / idx hold its reportable candidates in descending make_best_key
// order as end_strand / candidate index.  Walk them in that order and admit a candidate when it is distinct_alignment (candidate first,
// admitted alignment second) from every one admitted before; stop after k admissions (k = 0: none).  The admitted ones are compacted in
// place to the front of es / idx (entry m is written only after entry i >= m was read); returns their number.
__host__ __device__ inline uint32_t select_distinct(unsigned long long* es, uint32_t* idx, uint32_t n, uint32_t len, uint32_t k)
{
    uint32_t m = 0;
    for (uint32_t i = 0; i < n && (k == 0u || m < k); ++i) {
        const unsigned long long c = es[i];
        const uint32_t p = (uint32_t)(c >> 1), t = (uint32_t)(c & 1u);
        bool ok = true;
        for (uint32_t a = 0; a < m && ok; ++a) ok = distinct_alignment(p, t, (uint32_t)(es[a] >> 1), (uint32_t)(es[a] & 1u), len);
        if (!ok) continue;
        const uint32_t j = idx[i];
        es[m] = c; idx[m] = j; ++m;
    }
    return m;
}

// begin of an alignment ending at `end` of a read of length len: end - len, clamped at 0 (no traceback: soft clips and indels ignored)
__host__ __device__ __forceinline__ uint32_t aln_begin(uint32_t end, uint32_t len) { return end > len ? end - len : 0u; }

// ---------------------------------------------------------------------------------------------
// Paired-end policy (nvb_pair_params.policy / flags).  nvBowtie numbers its io::PE_POLICY_* FF 0, FR 1, RF 2, RR 3
// (nvbio/io/sequence/sequence.h:192-195); the C ABI numbers them NVB_PE_FR 0, NVB_PE_RF 1, NVB_PE_FF 2, NVB_PE_RR 3, so that a zeroed
// nvb_pair_params keeps the FR pairing:  NVB_PE_FR -> PE_POLICY_FR, NVB_PE_RF -> PE_POLICY_RF, NVB_PE_FF -> PE_POLICY_FF,
// NVB_PE_RR -> PE_POLICY_RR.
// ---------------------------------------------------------------------------------------------
struct PeFrame { bool left; uint32_t strand; };     // the other mate lies to the LEFT of the anchor; the strand it aligns on

// where the other mate of anchor mate a (0 = mate 1) aligned on strand t (0 forward) lies: nvBowtie's frame_opposite_mate
// (nvBowtie/bowtie2/cuda/alignment_utils.h:61-98) with anchor_fw = (t == 0)
__host__ __device__ __forceinline__ PeFrame pe_frame(uint32_t policy, uint32_t a, uint32_t t)
{
    const bool a1 = a == 0u, fw = t == 0u;
    bool left, ofw;
    switch (policy) {
    case NVB_PE_FF: left = a1 != fw; ofw = fw;  break;
    case NVB_PE_RR: left = a1 == fw; ofw = fw;  break;
    case NVB_PE_RF: left = fw;       ofw = !fw; break;
    default:        left = !fw;      ofw = !fw; break;      // NVB_PE_FR
    }
    PeFrame f; f.left = left; f.strand = ofw ? 0u : 1u;
    return f;
}

// Concordance of mate 1 (strand t1, [b1, e1)) and mate 2 (t2, [b2, e2)) under policy / flags: mate 2 lies on the strand the framing of
// mate 1 gives it, and with L / R the left / right mate as framed, L starts and ends no later than R, the fragment [L.b, R.e) is
// non-empty with a length in [min_frag, max_frag], and with NVB_PE_NO_OVERLAP L ends no later than R begins.  Framing from mate 2 gives
// the same answer.  NVB_PE_FR with flags 0: the forward mate is L (nvb_seed_extend_paired's original FR test).
__host__ __device__ __forceinline__ bool pe_concordant(uint32_t policy, uint32_t flags, uint32_t t1, uint32_t b1, uint32_t e1,
                                                       uint32_t t2, uint32_t b2, uint32_t e2, uint32_t min_frag, uint32_t max_frag)
{
    const PeFrame f = pe_frame(policy, 0u, t1);
    if (t2 != f.strand) return false;
    const uint32_t lb = f.left ? b2 : b1, le = f.left ? e2 : e1, rb = f.left ? b1 : b2, re = f.left ? e1 : e2;
    return lb <= rb && le <= re && re > lb && (re - lb) >= min_frag && (re - lb) <= max_frag && (!(flags & NVB_PE_NO_OVERLAP) || le <= rb);
}

// The opposite-mate window of anchor mate a aligned on strand t at [b, e): right of the anchor [b, min(b + max_frag, genome_len)),
// starting at e with NVB_PE_NO_OVERLAP; left of it [max(e - max_frag, 0), e), ending at b with NVB_PE_NO_OVERLAP
// (score_opposite_inl.h:177-193 without its min_frag trim).  Writes the window begin and length (0: empty) and returns the other mate's
// strand.
__host__ __device__ __forceinline__ uint32_t pe_rescue_window(uint32_t policy, uint32_t flags, uint32_t a, uint32_t t, uint32_t b, uint32_t e,
                                                              uint32_t max_frag, uint32_t genome_len, uint32_t& wb, uint32_t& wl)
{
    const PeFrame f = pe_frame(policy, a, t);
    const bool no_overlap = (flags & NVB_PE_NO_OVERLAP) != 0u;
    uint32_t we;
    if (f.left) { wb = e > max_frag ? e - max_frag : 0u; we = no_overlap ? b : e; }
    else        { wb = no_overlap ? e : b; we = (genome_len - b) < max_frag ? genome_len : b + max_frag; }
    wl = we > wb ? we - wb : 0u;
    return f.strand;
}

// ---------------------------------------------------------------------------------------------
// Second-best pair of nvb_seed_extend_paired_mapq.  A candidate pair is one alignment of each mate (end, strand, tie index); it is not
// distinct from the reported pair P* when BOTH its mates fail distinct_alignment against P*'s matching mate.  The second-best pair is
// the distinct candidate pair with the largest score, ties to the smaller mate-1 tie index, then the smaller mate-2 tie index -- a total
// order, so the answer does not depend on the order the candidates are offered in.
// ---------------------------------------------------------------------------------------------
struct PairSecond {
    uint32_t star_end[2], star_strand[2], len[2];              // P* and the mates' read lengths
    bool has; int32_t score; uint32_t end[2], strand[2], tie[2];

    __host__ __device__ __forceinline__ void init(uint32_t e1, uint32_t t1, uint32_t l1, uint32_t e2, uint32_t t2, uint32_t l2)
    {
        star_end[0] = e1; star_strand[0] = t1; len[0] = l1; star_end[1] = e2; star_strand[1] = t2; len[1] = l2;
        has = false; score = INT_MIN; end[0] = end[1] = 0xFFFFFFFFu; strand[0] = strand[1] = 0u; tie[0] = tie[1] = 0xFFFFFFFFu;
    }
    __host__ __device__ __forceinline__ void offer(int32_t s, uint32_t e1, uint32_t t1, uint32_t i1, uint32_t e2, uint32_t t2, uint32_t i2)
    {
        if (!distinct_alignment(e1, t1, star_end[0], star_strand[0], len[0]) && !distinct_alignment(e2, t2, star_end[1], star_strand[1], len[1]))
            return;
        if (has && (s < score || (s == score && (i1 > tie[0] || (i1 == tie[0] && i2 >= tie[1]))))) return;
        has = true; score = s; end[0] = e1; strand[0] = t1; tie[0] = i1; end[1] = e2; strand[1] = t2; tie[1] = i2;
    }
    // a rescue: anchor mate a's single-end best (end ae, strand at, tie index ai) with the other mate placed at end oe on strand ot, the
    // strand the policy frames it on (tie index 0xFFFFFFFF); s = the anchor's score + the rescue's
    __host__ __device__ __forceinline__ void offer_rescue(int a, int32_t s, uint32_t ae, uint32_t at, uint32_t ai, uint32_t oe, uint32_t ot)
    {
        if (a == 0) offer(s, ae, at, ai, oe, ot, 0xFFFFFFFFu);
        else        offer(s, oe, ot, 0xFFFFFFFFu, ae, at, ai);
    }
    // ... under NVB_PE_FR: the other mate on the anchor's opposite strand
    __host__ __device__ __forceinline__ void offer_rescue(int a, int32_t s, uint32_t ae, uint32_t at, uint32_t ai, uint32_t oe)
    {
        offer_rescue(a, s, ae, at, ai, oe, 1u - at);
    }
};

// a mate's candidates, merged per (strand, end) and sorted: the forward ones [0, n_fw), then the reverse ones [n_fw, n), each by end
struct MateCands { const uint32_t* end; const int32_t* score; const uint32_t* tie; uint32_t n_fw, n, len; };

// first index in [lo, hi) whose end is >= v
__host__ __device__ __forceinline__ uint32_t lower_bound_end(const uint32_t* end, uint32_t lo, uint32_t hi, uint64_t v)
{
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint64_t)end[mid] < v) lo = mid + 1; else hi = mid; }
    return lo;
}

// offer every concordant combination (pe_concordant) of one candidate of each mate.  Each candidate c of either mate is framed
// (pe_frame); when the other mate would lie to its left, c is skipped (that pair is visited from the other member), otherwise only the
// other mate's candidates on the framed strand ending in [c.begin + min_frag, c.begin + max_frag] are visited (binary search).  So every
// concordant combination is offered exactly once, and the work is bounded by the concordant combinations, not by the product of the
// two lists.  NVB_PE_FR: the forward candidates of either mate against the other mate's reverse ones.
__host__ __device__ inline void pair_combinations(const MateCands m[2], uint32_t policy, uint32_t flags, uint32_t min_frag, uint32_t max_frag,
                                                  PairSecond& ps)
{
    for (int a = 0; a < 2; ++a) {
        const MateCands& A = m[a]; const MateCands& B = m[1 - a];
        for (uint32_t t = 0; t < 2u; ++t) {
            const PeFrame f = pe_frame(policy, (uint32_t)a, t);
            if (f.left) continue;
            const uint32_t i0 = t ? A.n_fw : 0u, i1 = t ? A.n : A.n_fw, k0 = f.strand ? B.n_fw : 0u, k1 = f.strand ? B.n : B.n_fw;
            for (uint32_t i = i0; i < i1; ++i) {
                const uint32_t ae = A.end[i], ab = aln_begin(ae, A.len);
                uint32_t k = lower_bound_end(B.end, k0, k1, (uint64_t)ab + min_frag);
                for (; k < k1 && (uint64_t)B.end[k] <= (uint64_t)ab + max_frag; ++k) {
                    const uint32_t be = B.end[k], bb = aln_begin(be, B.len);
                    const bool ok = a == 0 ? pe_concordant(policy, flags, t, ab, ae, f.strand, bb, be, min_frag, max_frag)
                                           : pe_concordant(policy, flags, f.strand, bb, be, t, ab, ae, min_frag, max_frag);
                    if (!ok) continue;
                    const int32_t s = A.score[i] + B.score[k];
                    if (a == 0) ps.offer(s, ae, t, A.tie[i], be, f.strand, B.tie[k]);
                    else        ps.offer(s, be, f.strand, B.tie[k], ae, t, A.tie[i]);
                }
            }
        }
    }
}
// ... under NVB_PE_FR with flags 0
__host__ __device__ inline void pair_combinations(const MateCands m[2], uint32_t min_frag, uint32_t max_frag, PairSecond& ps)
{
    pair_combinations(m, NVB_PE_FR, 0u, min_frag, max_frag, ps);
}

// Mapping quality of an unpaired read: nvBowtie's BowtieMapq2 (mapq.h:155-327) for a scheme with perfect_score(len) = perfect,
// min_score(len) = min_score and m_monotone = monotone (match bonus 0, end-to-end).  The same float operations in the same order (only
// multiplies, subtractions, fabsf and compares: nothing the compiler could contract into an FMA), so host and device agree bit for bit.
// A read without an alignment (best = INT_MIN) is below any min_score > INT_MIN and gets 0.
__host__ __device__ inline uint32_t bowtie_mapq2(int32_t best_score, bool has_second, int32_t second_score, int32_t perfect, int32_t min_score,
                                                 bool monotone)
{
    const float max_s = (float)perfect, min_s = (float)min_score;
    const float diff = max_s - min_s;
    const float best = (float)best_score;
    if (best < min_s) return 0;
    const float best_over = best - min_s;
    const bool top = best_over == diff;
    if (monotone) {                                             // end-to-end
        if (!has_second) {
            if      (best_over >= diff * 0.8f) return 42;
            else if (best_over >= diff * 0.7f) return 40;
            else if (best_over >= diff * 0.6f) return 24;
            else if (best_over >= diff * 0.5f) return 23;
            else if (best_over >= diff * 0.4f) return 8;
            else if (best_over >= diff * 0.3f) return 3;
            return 0;
        }
        const float best_diff = fabsf(fabsf(best) - fabsf((float)second_score));
        if      (best_diff >= diff * 0.9f) return top ? 39 : 33;
        else if (best_diff >= diff * 0.8f) return top ? 38 : 27;
        else if (best_diff >= diff * 0.7f) return top ? 37 : 26;
        else if (best_diff >= diff * 0.6f) return top ? 36 : 22;
        else if (best_diff >= diff * 0.5f) return top ? 35 : best_over >= diff * 0.84f ? 25 : best_over >= diff * 0.68f ? 16 : 5;
        else if (best_diff >= diff * 0.4f) return top ? 34 : best_over >= diff * 0.84f ? 21 : best_over >= diff * 0.68f ? 14 : 4;
        else if (best_diff >= diff * 0.3f) return top ? 32 : best_over >= diff * 0.88f ? 18 : best_over >= diff * 0.67f ? 15 : 3;
        else if (best_diff >= diff * 0.2f) return top ? 31 : best_over >= diff * 0.88f ? 17 : best_over >= diff * 0.67f ? 11 : 0;
        else if (best_diff >= diff * 0.1f) return top ? 30 : best_over >= diff * 0.88f ? 12 : best_over >= diff * 0.67f ? 7 : 0;
        else if (best_diff > 0.0f)         return best_over >= diff * 0.67f ? 6 : 2;
        return best_over >= diff * 0.67f ? 1 : 0;
    }
    if (!has_second) {                                          // local
        if      (best_over >= diff * 0.8f) return 44;
        else if (best_over >= diff * 0.7f) return 42;
        else if (best_over >= diff * 0.6f) return 41;
        else if (best_over >= diff * 0.5f) return 36;
        else if (best_over >= diff * 0.4f) return 28;
        else if (best_over >= diff * 0.3f) return 24;
        return 22;
    }
    const float best_diff = fabsf(fabsf(best) - fabsf((float)second_score));
    if      (best_diff >= diff * 0.9f) return 40;
    else if (best_diff >= diff * 0.8f) return 39;
    else if (best_diff >= diff * 0.7f) return 38;
    else if (best_diff >= diff * 0.6f) return 37;
    else if (best_diff >= diff * 0.5f) return top ? 35 : best_over >= diff * 0.5f ? 25 : 20;
    else if (best_diff >= diff * 0.4f) return top ? 34 : best_over >= diff * 0.5f ? 21 : 19;
    else if (best_diff >= diff * 0.3f) return top ? 33 : best_over >= diff * 0.5f ? 18 : 16;
    else if (best_diff >= diff * 0.2f) return top ? 32 : best_over >= diff * 0.5f ? 17 : 12;
    else if (best_diff >= diff * 0.1f) return top ? 31 : best_over >= diff * 0.5f ? 14 : 9;
    else if (best_diff > 0.0f)         return best_over >= diff * 0.5f ? 11 : 2;
    return best_over >= diff * 0.5f ? 1 : 0;
}

// Window cut of a full-matrix traceback from a known sink (gotoh_full_warp_traceback_kernel): the first 0-based text row r0 it computes;
// it computes rows [r0, sink_x) and leaves the rest out.  Rows after sink_x cannot change a cell of rows <= sink_x (every type).  LOCAL
// with every gap charge < 0 (go, ge: the pattern gap open / extension gotoh_full_impl2 charges along both axes): an alignment of score
// `score` ending in pattern column sink_y consumes at most sink_y text symbols on substitutions (each worth <= s_max, the largest
// substitution score over all qualities) and, since a run of k deletions costs go + (k - 1) ge <= k max(go, ge) and insertions cost < 0,
// at most D_max = floor((sink_y s_max - score) / -max(go, ge)) on deletions; its source row is therefore >= sink_x - (sink_y + D_max).
// Starting from a zero row at r0 - 1 instead of the full rows above only lowers H / E / F (the recurrence is monotone and LOCAL's H >= 0),
// while every cell of the reference path keeps its value (its own path starts at or below r0); so at each cell of the path the set of
// maximal candidates can only shrink around the one the walk follows, and the walk retraces the same cells, ops and source.
__host__ __device__ inline uint32_t full_traceback_first_row(int type, uint32_t sink_x, uint32_t sink_y, int32_t score, int32_t s_max,
                                                             int32_t go, int32_t ge)
{
    if (type != NVB_LOCAL || go >= 0 || ge >= 0) return 0u;
    const int64_t g = go > ge ? go : ge;                                         // the most a deleted text symbol can cost (< 0)
    const int64_t room = (int64_t)sink_y * (s_max > 0 ? s_max : 0) - (int64_t)score;
    const int64_t span = (int64_t)sink_y + (room > 0 ? room / -g : 0);             // text symbols an alignment ending at the sink can consume
    return span < (int64_t)sink_x ? (uint32_t)((int64_t)sink_x - span) : 0u;
}

} // namespace nvb
