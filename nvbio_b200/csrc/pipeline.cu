// pipeline.cu -- seed + extend composition of the two hot paths (the loop nvbio's examples/fmmap/fmmap.cu:255-400
// and nvBowtie's best_approx run per read batch):
//
//   reads -> [fw, rc] strings -> seeds every `seed_interval` -> FM-index match (SA ranges)
//         -> locate every hit row -> diagonal -> genome window [diag - B/2, + read_len + B)
//         -> banded Gotoh score of the read (or its reverse complement) against the window
//         -> best score per read.
//
// Everything stays on the device between stages; the hit count never visits the host (the extension
// kernels read it from device memory).  Window rule: fmmap.cu:190-208 (genome_infixes); best-per-read
// reduction: fmmap.cu:365-385.
#include "fm_core.cuh"
#include "gotoh_core.cuh"
#include "pipeline_core.cuh"
#include "gotoh_full_core.cuh"
#include <cub/agent/single_pass_scan_operators.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <mutex>

namespace nvb {

struct PipeGeom {
    uint32_t n_reads;        // input reads
    uint32_t n_strings;      // n_reads * (both_strands ? 2 : 1)
    uint32_t strands;        // 1 or 2
    uint32_t stride;         // symbols per string slot in the [fw,rc] stream (multiple of 32/bits)
    uint32_t bits;           // symbol width of the [fw,rc] stream (= input width)
    uint32_t seeds_per_string;
    uint32_t seed_len, seed_interval;
    uint32_t band;
    uint32_t max_seed_hits;
    uint32_t genome_len;
};

// string s = 2*read + strand (strands==2) or read: copy / reverse-complement into an aligned slot.
// One thread per output word.
template <int BITS>
__global__ void __launch_bounds__(256)
pipe_make_strings_kernel(const StrSet reads, const PipeGeom g, uint32_t* __restrict__ out_words, uint32_t* __restrict__ out_len)
{
    constexpr uint32_t SPW = 32 / BITS;
    const uint32_t words_per_string = g.stride / SPW;
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= (uint64_t)g.n_strings * words_per_string) return;
    const uint32_t s = (uint32_t)(t / words_per_string), w = (uint32_t)(t % words_per_string);
    const uint32_t read = s / g.strands, strand = s % g.strands;
    const uint32_t off = str_off(reads, read), len = str_len(reads, read);
    if (w == 0) out_len[s] = len;
    uint32_t word = 0;
    for (uint32_t k = 0; k < SPW; ++k) {
        const uint32_t p = w * SPW + k;
        uint32_t c = 0;
        if (p < len) {
            if (strand == 0) c = sym_at_rt(reads.words, reads.bits, reads.big_endian, off + p);
            else { c = sym_at_rt(reads.words, reads.bits, reads.big_endian, off + (len - 1u - p)); c = (c < 4u) ? 3u - c : c; }
        }
        word |= c << (32u - BITS - BITS * k);              // big-endian packing
    }
    out_words[t] = word;
}

// base qualities of the [fw, rc] strings: byte p of string s at out[s * stride + p] (the rc string's are the read's, reversed)
__global__ void __launch_bounds__(256)
pipe_make_quals_kernel(const StrSet reads, const PipeGeom g, const uint8_t* __restrict__ quals, uint8_t* __restrict__ out)
{
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= (uint64_t)g.n_strings * g.stride) return;
    const uint32_t s = (uint32_t)(t / g.stride), p = (uint32_t)(t % g.stride);
    const uint32_t read = s / g.strands, strand = s % g.strands;
    const uint32_t off = str_off(reads, read), len = str_len(reads, read);
    out[t] = (p < len) ? quals[off + (strand == 0 ? p : len - 1u - p)] : (uint8_t)0;
}

// 2-bit fast path of the above: whole words at a time.  16 consecutive symbols starting at any symbol offset are a
// funnel shift of two words; the reverse complement of a word is ~brev(word) with the two bits of every symbol
// swapped back.
__device__ __forceinline__ uint32_t load16_2bit_be(const uint32_t* __restrict__ words, uint32_t p /* symbol offset */, uint32_t cnt /* symbols needed */)
{
    const uint32_t w = p >> 4, sh = 2u * (p & 15u);
    const uint32_t a = words[w];
    if (sh == 0) return a;
    const uint32_t b = ((p & 15u) + cnt > 16u) ? words[w + 1] : 0u;     // never touch a word the string does not reach
    return (a << sh) | (b >> (32u - sh));
}
__device__ __forceinline__ uint32_t revcomp16_2bit(uint32_t x)
{
    uint32_t y = __brev(~x);                                  // symbols reversed, bits inside each symbol swapped
    return ((y >> 1) & 0x55555555u) | ((y & 0x55555555u) << 1);
}
__global__ void __launch_bounds__(256)
pipe_make_strings_2bit_be_kernel(const StrSet reads, const PipeGeom g, uint32_t* __restrict__ out_words, uint32_t* __restrict__ out_len)
{
    const uint32_t words_per_string = g.stride / 16u;
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x, total = (uint64_t)g.n_strings * words_per_string;
    if (t >= total) return;
    // 32-bit index arithmetic whenever the word count allows it
    uint32_t s, w;
    if (total <= 0xFFFFFFFFull) { s = (uint32_t)t / words_per_string; w = (uint32_t)t - s * words_per_string; }
    else                        { s = (uint32_t)(t / words_per_string); w = (uint32_t)(t % words_per_string); }
    const uint32_t read = s / g.strands, strand = s % g.strands;
    const uint32_t off = str_off(reads, read), len = str_len(reads, read);
    if (w == 0) out_len[s] = len;
    const uint32_t first = w * 16u;                           // first output symbol of this word
    uint32_t word = 0;
    if (first < len) {
        const uint32_t cnt = (len - first) < 16u ? (len - first) : 16u;
        if (strand == 0) {
            word = load16_2bit_be(reads.words, off + first, cnt);
        } else {
            // output symbols first..first+cnt-1 are the complements of input symbols len-1-first .. len-first-cnt (descending)
            const uint32_t lo = len - first - cnt;            // lowest input symbol needed
            uint32_t x = load16_2bit_be(reads.words, off + lo, cnt);   // symbols lo .. lo+15 (only the first cnt matter)
            x = revcomp16_2bit(x);                             // now symbol (lo+15-j) sits at position j
            word = x << (2u * (16u - cnt));                    // drop the 16-cnt leading junk symbols
        }
        if (cnt < 16u) word &= ~(0xFFFFFFFFu >> (2u * cnt));   // zero the padding
    }
    out_words[t] = word;
}

// hits of a seed's SA range, clamped; y == 0xFFFFFFFF: one hit, already located (fm_match_locate_one)
__device__ __forceinline__ uint32_t seed_range_hits(uint2 range, uint32_t max_seed_hits)
{
    const uint32_t sz = (range.y == 0xFFFFFFFFu) ? 1u : ((range.x <= range.y) ? (range.y - range.x + 1u) : 0u);
    return sz < max_seed_hits ? sz : max_seed_hits;
}

// genome window [gb, ge) of a hit at text position pos of the seed at read offset seed_begin (fmmap.cu:198-199)
__device__ __forceinline__ uint2 hit_window(uint32_t pos, uint32_t seed_begin, uint32_t len, const PipeGeom& g)
{
    const uint32_t diag = pos > seed_begin ? pos - seed_begin : 0u;               // text position of read offset 0
    const uint32_t gb = diag > g.band / 2u ? diag - g.band / 2u : 0u;
    const uint64_t ge64 = (uint64_t)gb + len + g.band;
    return make_uint2(gb, ge64 < g.genome_len ? (uint32_t)ge64 : g.genome_len);
}

// one thread per (string, seed slot): SA range of the seed, and its clamped size (sizes == NULL on the per-read path, which sums the
// sizes of a read's ranges itself).
// genome != NULL (the per-read path on an index with the full suffix array): single-row ranges are located on the spot --
// ranges[q] = (text position, 0xFFFFFFFF), see fm_match_locate_one -- so that neither the remaining LF steps nor the later SA
// gather of that hit are needed; wider ranges stay SA ranges.
// (2048 threads per SM = every warp slot: the kernel lives on gathers in flight, so the register budget is 32)
// CTA size: seeds finish after 1 to 6 gathers, and a CTA's warp slots are only handed on when its last warp is done -- small CTAs
// keep more of the 64 slots busy
constexpr uint32_t SEED_BLOCK = 128;
constexpr uint32_t SEED_TODO_LISTS = 64;                     // todo lists (and counters) of the two-pass seed match
constexpr uint32_t SEED_TODO_PITCH = 32;                     // words between two counters: one 128-byte line each
constexpr uint32_t SEED_ITER = 8;                            // seeds per thread in its first pass
// DEFER: a seed whose k-mer occurs three or more times needs ~6 dependent gathers where the others need 1 to 3, and a warp's slot is
// held until its slowest lane is done -- such seeds are only looked up here (ranges[q] = the k-mer's range) and appended to `todo`;
// pipe_seed_match_wide_kernel finishes them, all lanes of its warps equally deep
template <int BITS, bool DEFER>
__global__ void __launch_bounds__(SEED_BLOCK, 2048 / SEED_BLOCK)
pipe_seed_match_kernel(const FmIndex f, const PipeGeom g, const uint32_t* __restrict__ words, const uint32_t* __restrict__ slen,
                       const uint32_t* __restrict__ genome, uint2* __restrict__ ranges, uint32_t* __restrict__ sizes,
                       uint32_t* __restrict__ todo, uint32_t* __restrict__ todo_count)
{
    // DEFER: SEED_ITER consecutive chunks of seeds per CTA (its seeds are done after one or two gathers: fewer, longer-lived CTAs; on its
    // own this measured no difference -- what bounded the first version of this pass was its atomics, see below)
    constexpr uint32_t ITER = DEFER ? SEED_ITER : 1u;
#pragma unroll 1
    for (uint32_t it = 0; it < ITER; ++it) {
        const uint32_t q = (blockIdx.x * ITER + it) * SEED_BLOCK + threadIdx.x;
        const bool live = q < g.n_strings * g.seeds_per_string;
        if (!DEFER && !live) return;
        uint32_t x = 1, y = 0;
        bool deferred = false;
        if (live) {
            const uint32_t s = q / g.seeds_per_string, k = q % g.seeds_per_string;
            const uint32_t len = slen[s];
            const uint32_t pos = k * g.seed_interval;
            if (pos + g.seed_len <= len) {
                if (genome) {
                    const uint32_t st = fm_match_locate_one<BITS, true, DEFER ? FM_DEFER : FM_WHOLE>(f, genome, words, s * g.stride + pos, g.seed_len, x, y);
                    if (st == FM_EMPTY) { x = 1; y = 0; }
                    deferred = DEFER && st == FM_DEFERRED;
                } else
                    fm_match_one<BITS, true>(f, words, s * g.stride + pos, g.seed_len, 0u, x, y);
            }
            ranges[q] = make_uint2(x, y);
            if (sizes && !deferred) sizes[q] = seed_range_hits(make_uint2(x, y), g.max_seed_hits);
        }
        if (DEFER) {
            // one atomic per warp, spread over SEED_TODO_LISTS counters, each in its own 128-byte line: same-line atomics serialise
            // in the L2.  List c takes the CTAs with blockIdx % LISTS == c, so its
            // capacity ceil(gridDim / LISTS) * SEED_BLOCK * SEED_ITER can never overflow
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, deferred);
            if (m) {
                const uint32_t lane = threadIdx.x & 31u, list = blockIdx.x % SEED_TODO_LISTS;
                const uint32_t cap = ((gridDim.x + SEED_TODO_LISTS - 1u) / SEED_TODO_LISTS) * SEED_BLOCK * SEED_ITER;
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(todo_count + list * SEED_TODO_PITCH, (uint32_t)__popc(m));
                base = __shfl_sync(0xFFFFFFFFu, base, 0);
                if (deferred) todo[(size_t)list * cap + base + __popc(m & ((1u << lane) - 1u))] = q;
            }
        }
    }
}
// the deferred seeds: resume from the k-mer's range.  CTA b works on list b % LISTS (gridDim is a multiple of LISTS), striding over it:
// the lists' lengths live on the device.  seed_grid = gridDim of the first pass (defines the lists' capacity)
template <int BITS>
__global__ void __launch_bounds__(SEED_BLOCK, 2048 / SEED_BLOCK)
pipe_seed_match_wide_kernel(const FmIndex f, const PipeGeom g, const uint32_t* __restrict__ words,
                            const uint32_t* __restrict__ genome, uint2* __restrict__ ranges, uint32_t* __restrict__ sizes,
                            const uint32_t* __restrict__ todo, const uint32_t* __restrict__ todo_count, const uint32_t seed_grid)
{
    const uint32_t list = blockIdx.x % SEED_TODO_LISTS, per_list = gridDim.x / SEED_TODO_LISTS;
    const uint32_t cap = ((seed_grid + SEED_TODO_LISTS - 1u) / SEED_TODO_LISTS) * SEED_BLOCK * SEED_ITER;
    const uint32_t n = todo_count[list * SEED_TODO_PITCH];
    for (uint32_t t = (blockIdx.x / SEED_TODO_LISTS) * SEED_BLOCK + threadIdx.x; t < n; t += per_list * SEED_BLOCK) {
        const uint32_t q = todo[(size_t)list * cap + t];
        const uint32_t s = q / g.seeds_per_string, k = q % g.seeds_per_string;
        const uint2 r = ranges[q];
        uint32_t x = r.x, y = r.y;
        if (fm_match_locate_one<BITS, true, FM_RESUME>(f, genome, words, s * g.stride + k * g.seed_interval, g.seed_len, x, y) == FM_EMPTY) { x = 1; y = 0; }
        ranges[q] = make_uint2(x, y);
        if (sizes) sizes[q] = seed_range_hits(make_uint2(x, y), g.max_seed_hits);
    }
}

__device__ __forceinline__ uint32_t upper_bound_u32(const uint32_t* __restrict__ a, uint32_t n, uint32_t v)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] <= v) lo = mid + 1; else hi = mid; }
    return lo;
}

// counts[0] = min(total, capacity), counts[1] = total
__global__ void pipe_count_kernel(const uint32_t* __restrict__ excl, const uint32_t* __restrict__ sizes, uint32_t n_queries, uint32_t capacity,
                                  uint32_t* __restrict__ counts)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const uint32_t total = n_queries ? excl[n_queries - 1] + sizes[n_queries - 1] : 0u;
        counts[1] = total;
        counts[0] = total < capacity ? total : capacity;
    }
}

// one thread per QUERY (most seeds have 0 or 1 hits): locate each of its SA rows, derive the genome window and the
// alignment job.  Hit h = excl[q] + j keeps the reference's slot order (filter_inl.h:99-118) without a binary search.
__global__ void __launch_bounds__(256)
pipe_expand_hits_kernel(const FmIndex f, const PipeGeom g, const uint2* __restrict__ ranges, const uint32_t* __restrict__ sizes,
                        const uint32_t* __restrict__ excl, const uint32_t* __restrict__ slen, const uint32_t* __restrict__ counts,
                        uint32_t* __restrict__ hit_string, uint32_t* __restrict__ p_off, uint32_t* __restrict__ p_len,
                        uint32_t* __restrict__ t_off, uint32_t* __restrict__ t_len)
{
    const uint32_t q = blockIdx.x * 256 + threadIdx.x;
    if (q >= g.n_strings * g.seeds_per_string) return;
    const uint32_t sz = sizes[q];
    if (sz == 0) return;
    const uint32_t base = excl[q], kept = counts[0];
    const uint32_t x = ranges[q].x;
    const uint32_t s = q / g.seeds_per_string, k = q % g.seeds_per_string;
    const uint32_t seed_begin = k * g.seed_interval;
    const uint32_t len = slen[s];
    for (uint32_t j = 0; j < sz; ++j) {
        const uint32_t h = base + j;
        if (h >= kept) break;                                                      // beyond the caller's capacity
        const uint2 w = hit_window(fm_locate_one(f, x + j), seed_begin, len, g);
        hit_string[h] = s;
        p_off[h] = s * g.stride; p_len[h] = len;
        t_off[h] = w.x;          t_len[h] = w.y - w.x;
    }
}

// ---------------------------------------------------------------------------------------------
// per-read path (no per-hit outputs requested): pipe_resolve_reads_kernel takes the seed ranges to the distinct (strand, window)
// alignment jobs of every read, their results where the exact shortcut proves them, and the best of those per read -- no per-seed
// size, no hit-slot scan and no per-hit array.  The jobs it leaves to the DP are scored after it; pipe_scatter_dp_kernel and
// pipe_finalize_dp_kernel then let a DP job replace a read's result when it beats the claimed best.  Job order varies from run to run,
// the results do not (every job carries the index of its first hit, and the best-per-read key breaks score ties by it exactly as the
// per-hit path breaks them by the hit index).
// ---------------------------------------------------------------------------------------------
struct Jobs { uint32_t *p_off, *p_len, *t_off, *t_len; };   // alignment jobs: a read string (offset, length) against a genome window

constexpr uint32_t RJ_BLOCK = 128;          // reads per tile (one CTA, one thread per read in phase A)
constexpr uint32_t RJ_STAGE = 640;          // staged jobs per CTA (average: ~1.2 per read); more go straight to the global lists
constexpr int      RJ_LOCAL = 6;            // distinct windows remembered per read (more are still scored, just not de-duplicated)
constexpr uint32_t RJ_CLAIMED = 0xFFFFFFFFu, RJ_CLAIMED_EMPTY = 0xFFFFFFFEu;   // st_slot of a job the shortcut resolved (else: DP slot)
using RjTileState = cub::ScanTileState<uint32_t>;
using RjPrefixOp  = cub::TilePrefixCallbackOp<uint32_t, ::cuda::std::plus<uint32_t>, RjTileState>;

// the tile states of the hit-slot look-back and the counters of one call, reset in stream order: counts[2] = jobs, counts[3] = tile ticket
__global__ void __launch_bounds__(256)
pipe_resolve_init_kernel(RjTileState tiles, const uint32_t n_tiles, uint32_t* __restrict__ counts, uint32_t* __restrict__ dp_count)
{
    tiles.InitializeStatus((int)n_tiles);
    if (blockIdx.x == 0 && threadIdx.x == 0) { counts[2] = 0u; counts[3] = 0u; *dp_count = 0u; }
}

// One tile of RJ_BLOCK reads per CTA.
//  * Hit slots: each read sums its clamped range sizes (its ranges are read from global memory: staging the tile's 28 KB of ranges in
//    shared memory measured 0.71 ms against 0.53 on the headline step: it cut the CTAs per SM from 7 to 5); a block scan plus a single-pass decoupled look-back over the tiles gives its first
//    slot (the per-hit path's exclusive scan at the read's first seed).  The tile index comes from a ticket, so every tile a CTA waits
//    on belongs to a CTA that is already running.  The last tile writes counts[0] = min(total, capacity), counts[1] = total.
//  * Phase A, one thread per read: locate, window and the RJ_LOCAL-window de-duplication (strands shared) of every kept hit
//    (slot < hit_capacity); jobs are staged in shared memory, a job that does not fit goes straight to the job list and the DP list.
//  * Phase B, the whole CTA over the staged jobs: append them to the job list (one atomic), run the exact shortcut (shortcut: 0 = off,
//    1 = with its one-gap check, 2 = without), compact the others into the DP list (one atomic) and reduce the claimed results per read
//    (64-bit make_best_key in shared memory).  Every read's best_key / score / end / strand is written here (none: 0 / INT_MIN /
//    0xFFFFFFFF / 0); a DP job replaces it later only with a larger key.
// 8 CTAs (32 warps) per SM, 64 registers, no spills: measured against 7 and 10 CTAs and against 64-read tiles at 14, 16 and 20 (DESIGN 5)
__global__ void __launch_bounds__(RJ_BLOCK, 8)
pipe_resolve_reads_kernel(const FmIndex f, const PipeGeom g, const uint2* __restrict__ ranges, const uint32_t* __restrict__ slen,
                          const uint32_t hit_capacity, RjTileState tiles, const uint32_t n_tiles, uint32_t* __restrict__ counts,
                          const int shortcut, const int32_t match, const int32_t mismatch, const int32_t max_gap_open,
                          const uint32_t* __restrict__ str_words, const uint32_t* __restrict__ genome,
                          uint32_t* __restrict__ j_string, uint32_t* __restrict__ j_first, const Jobs jobs,
                          int32_t* __restrict__ job_score, uint2* __restrict__ job_sink,
                          const Jobs dp, uint32_t* __restrict__ dp_job, uint32_t* __restrict__ dp_count,
                          unsigned long long* __restrict__ best_key, int32_t* best_score, uint32_t* best_pos, uint8_t* __restrict__ best_strand)
{
    using BlockScan = cub::BlockScan<uint32_t, RJ_BLOCK>;
    __shared__ struct { typename RjPrefixOp::TempStorage prefix; typename BlockScan::TempStorage scan; } s_tmp;
    __shared__ uint32_t st_string[RJ_STAGE], st_first[RJ_STAGE], st_toff[RJ_STAGE], st_tlen[RJ_STAGE], st_slot[RJ_STAGE];
    __shared__ unsigned long long s_key[RJ_BLOCK];
    __shared__ int32_t s_score[RJ_BLOCK];
    __shared__ uint32_t s_pos[RJ_BLOCK];
    __shared__ uint8_t s_strand[RJ_BLOCK];
    __shared__ uint32_t s_tile, s_cnt, s_base, s_dp_cnt, s_dp_base;
    if (threadIdx.x == 0) { s_tile = atomicAdd(counts + 3, 1u); s_cnt = 0u; s_dp_cnt = 0u; }
    s_key[threadIdx.x] = 0ull;
    __syncthreads();
    const uint32_t tile = s_tile, r0 = tile * RJ_BLOCK, r = r0 + threadIdx.x;
    const uint32_t per_read = g.strands * g.seeds_per_string;
    const bool live = r < g.n_reads;
    const uint2* rr = ranges + (size_t)r * per_read;            // this read's ranges: q = (r * strands + strand) * seeds + k

    // hit slots
    uint32_t hits = 0, run = 0;
    if (live)
        for (uint32_t q = 0; q < per_read; ++q) hits += seed_range_hits(rr[q], g.max_seed_hits);
    if (tile == 0) {
        uint32_t aggregate;
        BlockScan(s_tmp.scan).ExclusiveSum(hits, run, aggregate);
        if (threadIdx.x == 0) tiles.SetInclusive(0, aggregate);
    } else {
        RjPrefixOp prefix(tiles, s_tmp.prefix, ::cuda::std::plus<uint32_t>{}, (int)tile);
        BlockScan(s_tmp.scan).ExclusiveSum(hits, run, prefix);
    }
    if (tile == n_tiles - 1u && threadIdx.x == RJ_BLOCK - 1u) {  // dead threads add 0: the last thread's inclusive sum is the total
        const uint32_t total = run + hits;
        counts[1] = total;
        counts[0] = total < hit_capacity ? total : hit_capacity;
    }

    // phase A
    if (live) {
        uint32_t lk_s[RJ_LOCAL], lk_b[RJ_LOCAL], lk_e[RJ_LOCAL];
        int n_local = 0;
        for (uint32_t strand = 0; strand < g.strands; ++strand) {
            const uint32_t s = r * g.strands + strand;
            const uint32_t len = slen[s];
            for (uint32_t k = 0; k < g.seeds_per_string; ++k) {
                const uint2 rq = rr[strand * g.seeds_per_string + k];
                const bool located = rq.y == 0xFFFFFFFFu;                              // already a text position (fm_match_locate_one)
                const uint32_t sz = seed_range_hits(rq, g.max_seed_hits);
                if (sz == 0u) continue;
                const uint32_t base = run, x = rq.x, seed_begin = k * g.seed_interval;
                run += sz;
                for (uint32_t j = 0; j < sz; ++j) {
                    const uint32_t h = base + j;
                    if (h >= hit_capacity) break;                                      // beyond the caller's capacity
                    const uint2 w = hit_window(located ? x : fm_locate_one(f, x + j), seed_begin, len, g);
                    bool seen = false;
#pragma unroll
                    for (int e = 0; e < RJ_LOCAL; ++e) seen |= (e < n_local) && lk_s[e] == s && lk_b[e] == w.x && lk_e[e] == w.y;
                    if (seen) continue;
#pragma unroll
                    for (int e = 0; e < RJ_LOCAL; ++e) if (e == n_local) { lk_s[e] = s; lk_b[e] = w.x; lk_e[e] = w.y; }
                    if (n_local < RJ_LOCAL) ++n_local;
                    const uint32_t slot = atomicAdd(&s_cnt, 1u);
                    if (slot < RJ_STAGE) { st_string[slot] = s; st_first[slot] = h; st_toff[slot] = w.x; st_tlen[slot] = w.y - w.x; }
                    else {                                                             // staging full: straight to both global lists
                        const uint32_t o = atomicAdd(counts + 2, 1u), d = atomicAdd(dp_count, 1u);
                        j_string[o] = s; j_first[o] = h;
                        jobs.p_off[o] = s * g.stride; jobs.p_len[o] = len; jobs.t_off[o] = w.x; jobs.t_len[o] = w.y - w.x;
                        dp.p_off[d] = s * g.stride; dp.p_len[d] = len; dp.t_off[d] = w.x; dp.t_len[d] = w.y - w.x; dp_job[d] = o;
                    }
                }
            }
        }
    }
    __syncthreads();

    // phase B: job list, exact shortcut, claimed best per read
    const uint32_t n = s_cnt < RJ_STAGE ? s_cnt : RJ_STAGE;
    if (threadIdx.x == 0) s_base = n ? atomicAdd(counts + 2, n) : 0u;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += RJ_BLOCK) {
        const uint32_t o = s_base + i, s = st_string[i], first = st_first[i], len = slen[s], to = st_toff[i], N = st_tlen[i];
        j_string[o] = s; j_first[o] = first; jobs.p_off[o] = s * g.stride; jobs.p_len[o] = len; jobs.t_off[o] = to; jobs.t_len[o] = N;
        int32_t score = 0; uint32_t sx = 0, sy = 0;
        if (shortcut && gapless_job_shortcut(str_words, genome, s * g.stride, len, to, N, g.band, match, mismatch, max_gap_open, score, sx, sy,
                                             shortcut != 2)) {
            const uint2 sk = make_uint2(sx, sy);
            job_score[o] = score; job_sink[o] = sk;
            if (job_aligned(sk)) {
                st_slot[i] = RJ_CLAIMED; st_toff[i] = to + sx; st_tlen[i] = (uint32_t)score;   // (the DP list never reads a claimed job)
                atomicMax(&s_key[s / g.strands - r0], make_best_key(score, first));
            } else st_slot[i] = RJ_CLAIMED_EMPTY;
        } else st_slot[i] = atomicAdd(&s_dp_cnt, 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) s_dp_base = s_dp_cnt ? atomicAdd(dp_count, s_dp_cnt) : 0u;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += RJ_BLOCK) {
        const uint32_t slot = st_slot[i], s = st_string[i];
        if (slot == RJ_CLAIMED) {                                // the claimed job whose key won writes its read's result
            const uint32_t rl = s / g.strands - r0;
            const int32_t score = (int32_t)st_tlen[i];
            if (s_key[rl] == make_best_key(score, st_first[i])) { s_score[rl] = score; s_pos[rl] = st_toff[i]; s_strand[rl] = (uint8_t)(s % g.strands); }
        } else if (slot != RJ_CLAIMED_EMPTY) {
            const uint32_t d = s_dp_base + slot;
            dp.p_off[d] = s * g.stride; dp.p_len[d] = slen[s]; dp.t_off[d] = st_toff[i]; dp.t_len[d] = st_tlen[i]; dp_job[d] = s_base + i;
        }
    }
    __syncthreads();
    if (live) {
        const unsigned long long key = s_key[threadIdx.x];
        best_key[r] = key;
        best_score[r] = key ? s_score[threadIdx.x] : INT_MIN;
        best_pos[r] = key ? s_pos[threadIdx.x] : 0xFFFFFFFFu;
        best_strand[r] = key ? s_strand[threadIdx.x] : (uint8_t)0;
    }
}

// the DP's results back into the job list, and its aligned jobs into the best-per-read reduction
__global__ void __launch_bounds__(256)
pipe_scatter_dp_kernel(const PipeGeom g, const uint32_t* __restrict__ dp_count, const uint32_t* __restrict__ dp_job,
                       const int32_t* __restrict__ dp_score, const uint2* __restrict__ dp_sink,
                       const uint32_t* __restrict__ j_string, const uint32_t* __restrict__ j_first,
                       int32_t* __restrict__ job_score, uint2* __restrict__ job_sink, unsigned long long* __restrict__ best_key)
{
    const uint32_t n = *dp_count;
    for (uint32_t a = blockIdx.x * 256 + threadIdx.x; a < n; a += gridDim.x * 256) {
        const uint32_t j = dp_job[a];
        const int32_t sc = dp_score[a];
        const uint2 sk = dp_sink[a];
        job_score[j] = sc; job_sink[j] = sk;
        if (job_aligned(sk)) atomicMax(best_key + j_string[j] / g.strands, make_best_key(sc, j_first[j]));
    }
}

// a DP job whose key is its read's best key writes the read's result (first-hit indices are unique: at most one job of the read matches,
// and none does when a claimed job won -- that one already wrote it)
__global__ void __launch_bounds__(256)
pipe_finalize_dp_kernel(const PipeGeom g, const uint32_t* __restrict__ dp_count, const uint32_t* __restrict__ dp_job,
                        const int32_t* __restrict__ dp_score, const uint2* __restrict__ dp_sink, const uint32_t* __restrict__ dp_t_off,
                        const uint32_t* __restrict__ j_string, const uint32_t* __restrict__ j_first,
                        const unsigned long long* __restrict__ best_key,
                        int32_t* __restrict__ best_score, uint32_t* __restrict__ best_pos, uint8_t* __restrict__ best_strand)
{
    const uint32_t n = *dp_count;
    for (uint32_t a = blockIdx.x * 256 + threadIdx.x; a < n; a += gridDim.x * 256) {
        const uint32_t j = dp_job[a], s = j_string[j], read = s / g.strands;
        const int32_t sc = dp_score[a];
        if (best_key[read] != make_best_key(sc, j_first[j])) continue;
        best_score[read] = sc; best_pos[read] = dp_t_off[a] + dp_sink[a].x; best_strand[read] = (uint8_t)(s % g.strands);
    }
}

// Hits of one string are contiguous (queries are ordered by string, then seed).  Several seeds of a read usually
// vote for the same diagonal, i.e. the very same (string, window) alignment job: score it once.
// leader[h] = the smallest h' <= h of the same string with the same window; flag[h] = (leader[h] == h).
// A missed duplicate (beyond the look-back) only costs a redundant alignment, never a different result.
__global__ void __launch_bounds__(256)
pipe_find_leaders_kernel(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ hit_string,
                         const uint32_t* __restrict__ t_off, const uint32_t* __restrict__ t_len,
                         uint32_t* __restrict__ leader, uint32_t* __restrict__ flag)
{
    // the block's 256 hits plus the 64 before them, staged once in shared memory (the look-back re-reads them ~5x on average)
    constexpr uint32_t BACK = 64u;
    __shared__ uint32_t ss[256 + BACK], so[256 + BACK], sl[256 + BACK];
    const uint32_t n = counts[0];
    const uint32_t h0 = blockIdx.x * 256;
    if (h0 >= n) return;
    for (uint32_t i = threadIdx.x; i < 256 + BACK; i += 256) {
        const int64_t g = (int64_t)h0 - BACK + i;
        const bool in = g >= 0 && g < (int64_t)n;
        ss[i] = in ? hit_string[g] : 0xFFFFFFFFu; so[i] = in ? t_off[g] : 0u; sl[i] = in ? t_len[g] : 0u;
    }
    __syncthreads();
    const uint32_t h = h0 + threadIdx.x;
    if (h >= n) return;
    const uint32_t me = threadIdx.x + BACK;
    const uint32_t s = ss[me], o = so[me], l = sl[me];
    uint32_t lead = h;
    for (uint32_t back = 1; back <= BACK && back <= h; ++back) {
        if (ss[me - back] != s) break;
        if (so[me - back] == o && sl[me - back] == l) lead = h - back;
    }
    leader[h] = lead;
    flag[h] = (lead == h) ? 1u : 0u;
}

// counts[2] = number of unique jobs
__global__ void pipe_job_count_kernel(const uint32_t* __restrict__ job_idx, const uint32_t* __restrict__ flag, uint32_t* __restrict__ counts)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const uint32_t n = counts[0];
        counts[2] = n ? job_idx[n - 1] + flag[n - 1] : 0u;
    }
}

__global__ void __launch_bounds__(256)
pipe_compact_jobs_kernel(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ job_idx,
                         const uint32_t* __restrict__ p_off, const uint32_t* __restrict__ p_len,
                         const uint32_t* __restrict__ t_off, const uint32_t* __restrict__ t_len,
                         uint32_t* __restrict__ jp_off, uint32_t* __restrict__ jp_len, uint32_t* __restrict__ jt_off, uint32_t* __restrict__ jt_len)
{
    const uint32_t h = blockIdx.x * 256 + threadIdx.x;
    if (h >= counts[0] || !flag[h]) return;
    const uint32_t j = job_idx[h];
    jp_off[j] = p_off[h]; jp_len[j] = p_len[h]; jt_off[j] = t_off[h]; jt_len[j] = t_len[h];
}

// every hit receives its group's (score, sink); the best-per-read reduction (see pipe_reduce_kernel) rides along
__global__ void __launch_bounds__(256)
pipe_scatter_scores_kernel(const PipeGeom g, const uint32_t* __restrict__ counts, const uint32_t* __restrict__ leader, const uint32_t* __restrict__ job_idx,
                           const int32_t* __restrict__ job_score, const uint2* __restrict__ job_sink, const uint32_t* __restrict__ hit_string,
                           int32_t* __restrict__ score, uint2* __restrict__ sink, unsigned long long* __restrict__ best_key)
{
    const uint32_t h = blockIdx.x * 256 + threadIdx.x;
    if (h >= counts[0]) return;
    // leader[h] is the earliest identical job within the look-back of h; it may itself have an earlier one: follow the chain to
    // the hit that really was compacted into the job list (leader[l] == l)
    uint32_t l = leader[h];
    for (uint32_t nx = leader[l]; nx != l; nx = leader[l]) l = nx;
    const uint32_t j = job_idx[l];
    const int32_t sc = job_score[j];
    const uint2 sk = job_sink[j];
    score[h] = sc;
    sink[h]  = sk;
    if (job_aligned(sk)) atomicMax(best_key + hit_string[h] / g.strands, make_best_key(sc, h));
}

// best hit per read: max score, ties -> smallest hit index (deterministic)
__global__ void __launch_bounds__(256)
pipe_reduce_kernel(const PipeGeom g, const uint32_t* __restrict__ counts, const uint32_t* __restrict__ hit_string,
                   const int32_t* __restrict__ score, const uint2* __restrict__ sink, unsigned long long* __restrict__ best_key)
{
    const uint32_t h = blockIdx.x * 256 + threadIdx.x;
    if (h >= counts[0] || !job_aligned(sink[h])) return;
    atomicMax(best_key + hit_string[h] / g.strands, make_best_key(score[h], h));
}

__global__ void __launch_bounds__(256)
pipe_finalize_kernel(const PipeGeom g, const unsigned long long* __restrict__ best_key, const uint32_t* __restrict__ t_off,
                     const uint2* __restrict__ sink, const uint32_t* __restrict__ hit_string,
                     int32_t* __restrict__ best_score, uint32_t* __restrict__ best_pos, uint8_t* __restrict__ best_strand)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= g.n_reads) return;
    const unsigned long long key = best_key[r];
    if (key == 0ull) { best_score[r] = INT_MIN; best_pos[r] = 0xFFFFFFFFu; if (best_strand) best_strand[r] = 0; return; }
    const uint32_t h = best_key_index(key);
    best_score[r] = best_key_score(key);
    best_pos[r] = t_off[h] + sink[h].x;
    if (best_strand) best_strand[r] = (uint8_t)(hit_string[h] % g.strands);
}

// the best hit of every read as an alignment job for the traceback (reads without a hit get an empty job)
__global__ void __launch_bounds__(256)
pipe_best_jobs_kernel(const PipeGeom g, const unsigned long long* __restrict__ best_key, const uint32_t* __restrict__ hit_string,
                      const uint32_t* __restrict__ p_off, const uint32_t* __restrict__ p_len,
                      const uint32_t* __restrict__ t_off, const uint32_t* __restrict__ t_len,
                      uint32_t* __restrict__ bp_off, uint32_t* __restrict__ bp_len, uint32_t* __restrict__ bt_off, uint32_t* __restrict__ bt_len,
                      uint8_t* __restrict__ strand)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= g.n_reads) return;
    const unsigned long long key = best_key[r];
    if (key == 0ull) { bp_off[r] = 0; bp_len[r] = 0; bt_off[r] = 0; bt_len[r] = 0; if (strand) strand[r] = 0; return; }
    const uint32_t h = best_key_index(key);
    bp_off[r] = p_off[h]; bp_len[r] = p_len[h]; bt_off[r] = t_off[h]; bt_len[r] = t_len[h];
    if (strand) strand[r] = (uint8_t)(hit_string[h] % g.strands);
}

// The alignments the extension scored, as every later stage reads them: the per-read path's distinct jobs (tie index: the job's first
// hit) or the per-hit path's kept hits (tie == NULL: the hit itself).  Both paths see the same (score, strand, end, smallest tie index)
// set, so what is derived from it does not depend on the path, the job order or the de-duplication.  The count lives on the device.
struct Scored {
    const uint32_t* count; const uint32_t* string; const uint32_t* tie_index; Jobs jobs; const int32_t* score; const uint2* sink;
    __device__ __forceinline__ uint32_t tie(uint32_t j) const { return tie_index ? tie_index[j] : j; }
    __device__ __forceinline__ uint32_t end(uint32_t j) const { return jobs.t_off[j] + sink[j].x; }
};

// per-read path: the best job of every read as its traceback job (pipe_best_jobs_kernel's output).  pipe_empty_jobs_kernel first gives
// every read an empty job; pipe_winner_kernel then lets the best job write its own
__global__ void __launch_bounds__(256)
pipe_empty_jobs_kernel(const uint32_t n_reads, uint32_t* __restrict__ bp_off, uint32_t* __restrict__ bp_len, uint32_t* __restrict__ bt_off,
                       uint32_t* __restrict__ bt_len, uint8_t* __restrict__ strand)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= n_reads) return;
    bp_off[r] = 0; bp_len[r] = 0; bt_off[r] = 0; bt_len[r] = 0;
    if (strand) strand[r] = 0;
}

// the candidate whose make_best_key is its read's key writes the read's job, end and strand (each skipped when NULL); tie indices are
// unique, so at most one candidate of a read matches.  Resident grid striding over the device-side count
__global__ void __launch_bounds__(256)
pipe_winner_kernel(const PipeGeom g, const Scored c, const unsigned long long* __restrict__ key, const Jobs out,
                   uint32_t* __restrict__ end, uint8_t* __restrict__ strand)
{
    const uint32_t n = *c.count;
    for (uint32_t j = blockIdx.x * 256 + threadIdx.x; j < n; j += gridDim.x * 256) {
        const uint32_t s = c.string[j], r = s / g.strands;
        if (key[r] != make_best_key(c.score[j], c.tie(j))) continue;
        if (out.p_off) { out.p_off[r] = c.jobs.p_off[j]; out.p_len[r] = c.jobs.p_len[j]; out.t_off[r] = c.jobs.t_off[j]; out.t_len[r] = c.jobs.t_len[j]; }
        if (end) end[r] = c.end(j);
        if (strand) strand[r] = (uint8_t)(s % g.strands);
    }
}

// source cell (window-relative text start, read start) -> (genome coordinate, read start) of the first n traced jobs (d_n != NULL:
// *d_n).  best_key != NULL: job r is read r's best, and a read without a hit gets n_ops 0
__global__ void __launch_bounds__(256)
traceback_begin_kernel(const uint32_t* __restrict__ d_n, const uint32_t n, const unsigned long long* __restrict__ best_key,
                       const uint32_t* __restrict__ t_off, const uint2* __restrict__ source, uint32_t* __restrict__ n_ops, uint2* __restrict__ begin)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= (d_n ? *d_n : n)) return;
    if (best_key && best_key[i] == 0ull) { n_ops[i] = 0; begin[i] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu); return; }
    const uint2 sc = source[i];
    begin[i] = make_uint2(t_off[i] + sc.x, sc.y);
}

__global__ void __launch_bounds__(256)
pipe_export_hits_kernel(const PipeGeom g, const uint32_t* __restrict__ counts, const uint32_t* __restrict__ hit_string,
                        const uint32_t* __restrict__ t_off, const uint32_t* __restrict__ t_len,
                        uint32_t* __restrict__ out_read, uint2* __restrict__ out_window)
{
    const uint32_t h = blockIdx.x * 256 + threadIdx.x;
    if (h >= counts[0]) return;
    if (out_read)   out_read[h] = hit_string[h];              // string id = read*strands + strand
    if (out_window) out_window[h] = make_uint2(t_off[h], t_off[h] + t_len[h]);
}

// ---------------------------------------------------------------------------------------------
// second-best distinct alignment and MAPQ (nvb_seed_extend_mapq).  The candidates are the scored alignments of a read (Scored).
// ---------------------------------------------------------------------------------------------

// a candidate competes for the second-best alignment when it reaches the read's min score and is distinct from the best alignment
__device__ __forceinline__ bool second_candidate(int32_t score, uint32_t end, uint32_t strand, uint32_t len, uint32_t best_end,
                                                 uint32_t best_strand, const int32_t* __restrict__ min_score)
{
    return score >= min_score[len] && distinct_alignment(end, strand, best_end, best_strand, len);
}

// best qualifying candidate per read (64-bit atomicMax of make_best_key); resident grid striding over the device-side count
__global__ void __launch_bounds__(256)
pipe_second_reduce_kernel(const PipeGeom g, const Scored c, const uint32_t* __restrict__ str_len, const uint32_t* __restrict__ best_pos,
                          const uint8_t* __restrict__ best_strand, const int32_t* __restrict__ min_score,
                          unsigned long long* __restrict__ second_key)
{
    const uint32_t n = *c.count;
    for (uint32_t j = blockIdx.x * 256 + threadIdx.x; j < n; j += gridDim.x * 256) {
        const uint32_t s = c.string[j], read = s / g.strands;
        const int32_t sc = c.score[j];
        if (job_aligned(c.sink[j]) && second_candidate(sc, c.end(j), s % g.strands, str_len[s], best_pos[read], best_strand[read], min_score))
            atomicMax(second_key + read, make_best_key(sc, c.tie(j)));
    }
}

// one thread per read: the second score (INT_MIN / 0xFFFFFFFF / strand 0 when there is none) and BowtieMapq2
__global__ void __launch_bounds__(256)
pipe_mapq_kernel(const PipeGeom g, const nvb_mapq_params mp, const uint32_t* __restrict__ str_len, const int32_t* __restrict__ best_score,
                 const unsigned long long* __restrict__ second_key, int32_t* __restrict__ second_score, uint32_t* __restrict__ second_pos,
                 uint8_t* __restrict__ second_strand, uint8_t* __restrict__ mapq)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= g.n_reads) return;
    const unsigned long long key = second_key[r];
    const bool has = key != 0ull;
    const int32_t s2 = has ? best_key_score(key) : INT_MIN;
    second_score[r] = s2;
    if (!has) {
        if (second_pos) second_pos[r] = 0xFFFFFFFFu;
        if (second_strand) second_strand[r] = 0;
    }
    const uint32_t len = str_len[r * g.strands];
    mapq[r] = (uint8_t)bowtie_mapq2(best_score[r], has, s2, (int32_t)len * mp.match_bonus, mp.d_min_score[len], mp.match_bonus == 0);
}

// nvb_debug_mapq_eval: bowtie_mapq2 over arrays
__global__ void __launch_bounds__(256)
debug_mapq_eval_kernel(const int32_t* __restrict__ best, const uint8_t* __restrict__ has_second, const int32_t* __restrict__ second,
                       const uint32_t* __restrict__ len, const int32_t* __restrict__ match_bonus, const int32_t* __restrict__ min_score,
                       uint32_t n, uint8_t* __restrict__ mapq)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    mapq[i] = (uint8_t)bowtie_mapq2(best[i], has_second[i] != 0, second[i], (int32_t)len[i] * match_bonus[i], min_score[i], match_bonus[i] == 0);
}

// candidate segments of the paired MAPQ and of nvb_seed_extend_all (PipeCall::cand_segments): reportable candidates per read (counts) or
// their place in the read's segment (seg != NULL: cursor = counts zeroed, key = (strand << 32) | end, or ~make_best_key when by_best:
// ascending keys are then nvb_seed_extend_all's rank order)
__global__ void __launch_bounds__(256)
cand_scatter_kernel(const PipeGeom g, const Scored c, const uint32_t* __restrict__ str_len, const int32_t* __restrict__ min_score,
                    const uint32_t* __restrict__ seg, uint32_t* __restrict__ cursor, unsigned long long* __restrict__ key,
                    uint32_t* __restrict__ val, const bool by_best)
{
    const uint32_t n = *c.count;
    for (uint32_t j = blockIdx.x * 256 + threadIdx.x; j < n; j += gridDim.x * 256) {
        const uint32_t s = c.string[j], read = s / g.strands;
        if (!reportable(c.score[j], c.sink[j], min_score[str_len[s]])) continue;
        const uint32_t slot = atomicAdd(cursor + read, 1u);
        if (!seg) continue;
        key[seg[read] + slot] = by_best ? ~make_best_key(c.score[j], c.tie(j)) : ((unsigned long long)(s % g.strands) << 32) | c.end(j);
        val[seg[read] + slot] = j;
    }
}

// ---------------------------------------------------------------------------------------------
// up to k distinct alignments per read (nvb_seed_extend_all).  The candidate segments in rank order (descending make_best_key);
// all_select_kernel walks them (select_distinct), the exclusive scan of its counts is d_first, and all_emit_kernel writes the stored
// alignments and their traceback jobs, which are traced in slices of n_reads.
// ---------------------------------------------------------------------------------------------

// one thread per read: its sorted segment as end_strand (es, over the sorted keys), then select_distinct in place; cnt[r] = the read's
// alignments, their candidate indices at idx[seg[r] ..]
__global__ void __launch_bounds__(256)
all_select_kernel(const PipeGeom g, const Scored c, const uint32_t* __restrict__ str_len, const uint32_t* __restrict__ seg,
                  unsigned long long* __restrict__ es, uint32_t* __restrict__ idx, const uint32_t k, uint32_t* __restrict__ cnt)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= g.n_reads) return;
    const uint32_t b = seg[r], n = seg[r + 1] - b;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t j = idx[b + i];
        es[b + i] = end_strand(c.end(j), c.string[j] % g.strands);
    }
    cnt[r] = select_distinct(es + b, idx + b, n, str_len[r * g.strands], k);
}

// count = (alignments stored, wanted): the stored reads are the prefix with first[r + 1] <= capacity.  slice_n[t] = the stored alignments
// of traceback slice t, [t * n_reads, (t + 1) * n_reads)
__global__ void __launch_bounds__(256)
all_count_kernel(const uint32_t n_reads, const uint32_t* __restrict__ first, const uint32_t capacity, const uint32_t n_slices,
                 uint32_t* __restrict__ count, uint32_t* __restrict__ slice_n)
{
    const uint32_t stored = first[upper_bound_u32(first, n_reads + 1u, capacity) - 1u];   // first[0] = 0 <= capacity
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t == 0) { count[0] = stored; count[1] = first[n_reads]; }
    if (t >= n_slices) return;
    const uint64_t b = (uint64_t)t * n_reads;
    slice_n[t] = stored > b ? (uint32_t)(stored - b < n_reads ? stored - b : n_reads) : 0u;
}

// one thread per read whose alignments fit: alignment first[r] + i is its candidate idx[seg[r] + i]; its traceback job into `jobs`
__global__ void __launch_bounds__(256)
all_emit_kernel(const PipeGeom g, const Scored c, const uint32_t* __restrict__ first, const uint32_t* __restrict__ seg,
                const uint32_t* __restrict__ idx, const uint32_t capacity, uint32_t* __restrict__ out_read, int32_t* __restrict__ out_score,
                uint32_t* __restrict__ out_pos, uint8_t* __restrict__ out_strand, const Jobs jobs)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= g.n_reads) return;
    const uint32_t o = first[r], e = first[r + 1];
    if (e > capacity) return;
    const uint32_t* sel = idx + seg[r];
    for (uint32_t a = o; a < e; ++a) {
        const uint32_t j = sel[a - o], s = c.string[j];
        out_read[a] = r; out_score[a] = c.score[j]; out_pos[a] = c.end(j); out_strand[a] = (uint8_t)(s % g.strands);
        jobs.p_off[a] = c.jobs.p_off[j]; jobs.p_len[a] = c.jobs.p_len[j]; jobs.t_off[a] = c.jobs.t_off[j]; jobs.t_len[a] = c.jobs.t_len[j];
    }
}

// ---------------------------------------------------------------------------------------------
// paired-end stage (see nvb_seed_extend_paired in the header for the rules)
// ---------------------------------------------------------------------------------------------
struct MateBest { bool has; int32_t score; uint32_t strand, beg, end, len; };

// the best alignment of read r as the single-end stages left it: score, end (one past the last aligned base), strand
__device__ __forceinline__ MateBest mate_best(const PipeGeom& g, uint32_t r, const int32_t* best_score,
                                              const uint32_t* best_pos, const uint8_t* __restrict__ best_strand,
                                              const uint32_t* __restrict__ str_len)
{
    MateBest m; m.has = false; m.score = INT_MIN; m.strand = 0; m.beg = m.end = 0xFFFFFFFFu; m.len = 0;
    const uint32_t end = best_pos[r];
    if (end == 0xFFFFFFFFu) return m;
    m.has = true;
    m.score = best_score[r];
    m.strand = best_strand[r];
    m.len = str_len[r * g.strands];                 // both strands of a read have its length
    m.end = end;
    m.beg = aln_begin(m.end, m.len);
    return m;
}

// one thread per pair: concordance of the independent best alignments, else up to two opposite-mate jobs (slot 2p + anchor)
__global__ void __launch_bounds__(256)
pair_classify_kernel(const PipeGeom g, const uint32_t n_pairs, const nvb_pair_params pp,
                     // best_score / best_pos ARE mate_score / mate_pos in the paired entry point (the single-end stage writes the per-read
                     // bests straight into the mate arrays): no __restrict__ / const on either view
                     const int32_t* best_score, const uint32_t* best_pos, const uint8_t* __restrict__ best_strand,
                     const uint32_t* __restrict__ str_len,
                     uint32_t* __restrict__ want, uint32_t* __restrict__ w_pstr, uint32_t* __restrict__ w_toff, uint32_t* __restrict__ w_tlen,
                     int32_t* __restrict__ pair_score, uint32_t* __restrict__ pair_flags,
                     int32_t* mate_score, uint32_t* mate_pos, uint8_t* __restrict__ mate_strand)
{
    const uint32_t p = blockIdx.x * 256 + threadIdx.x;
    if (p >= n_pairs) return;
    MateBest m[2];
    m[0] = mate_best(g, p, best_score, best_pos, best_strand, str_len);
    m[1] = mate_best(g, n_pairs + p, best_score, best_pos, best_strand, str_len);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        mate_score[k * n_pairs + p] = m[k].score; mate_pos[k * n_pairs + p] = m[k].end; mate_strand[k * n_pairs + p] = (uint8_t)m[k].strand;
    }
    bool conc = m[0].has && m[1].has && (m[0].strand != m[1].strand);
    if (conc) {
        const MateBest& f = m[0].strand == 0 ? m[0] : m[1];
        const MateBest& r = m[0].strand == 0 ? m[1] : m[0];
        conc = fr_concordant(f.beg, f.end, r.beg, r.end, pp.min_frag, pp.max_frag);
    }
    if (conc) {
        pair_score[p] = m[0].score + m[1].score; pair_flags[p] = NVB_PAIR_CONCORDANT;
        want[2 * p] = want[2 * p + 1] = 0u;
        return;
    }
    pair_score[p] = INT_MIN; pair_flags[p] = NVB_PAIR_UNPAIRED;
#pragma unroll
    for (int a = 0; a < 2; ++a) {                               // a = anchor mate, 1 - a = the mate to place
        uint32_t w = 0u, ps = 0u, to = 0u, tl = 0u;
        if (m[a].has && m[a].score >= pp.min_mate_score) {
            const uint32_t o_read = (uint32_t)(1 - a) * n_pairs + p;
            if (m[a].strand == 0u) { to = m[a].beg; const uint32_t e = (g.genome_len - to) < pp.max_frag ? g.genome_len : to + pp.max_frag; tl = e - to; ps = 2u * o_read + 1u; }
            else                   { to = m[a].end > pp.max_frag ? m[a].end - pp.max_frag : 0u; tl = m[a].end - to; ps = 2u * o_read; }
            w = (tl >= 1u && str_len[ps] >= 1u) ? 1u : 0u;
        }
        want[2 * p + a] = w; w_pstr[2 * p + a] = ps; w_toff[2 * p + a] = to; w_tlen[2 * p + a] = tl;
    }
}

__global__ void __launch_bounds__(256)
pair_compact_kernel(const PipeGeom g, const uint32_t n_slots, const uint32_t capacity, const uint32_t* __restrict__ want, const uint32_t* __restrict__ job_idx,
                    const uint32_t* __restrict__ w_pstr, const uint32_t* __restrict__ w_toff, const uint32_t* __restrict__ w_tlen,
                    const uint32_t* __restrict__ str_len,
                    uint32_t* __restrict__ jp_off, uint32_t* __restrict__ jp_len, uint32_t* __restrict__ jt_off, uint32_t* __restrict__ jt_len)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n_slots || !want[i]) return;
    const uint32_t j = job_idx[i];
    if (j >= capacity) return;
    jp_off[j] = w_pstr[i] * g.stride; jp_len[j] = str_len[w_pstr[i]]; jt_off[j] = w_toff[i]; jt_len[j] = w_tlen[i];
}

// slot i = 2p + a (anchor a of pair p): whether its opposite-mate job was run (within the rescue capacity) and reached min_mate_score;
// if so, the rescued alignment's score and end
__device__ __forceinline__ bool usable_rescue(const nvb_pair_params& pp, const uint32_t* __restrict__ want, const uint32_t* __restrict__ job_idx,
                                              const uint32_t* __restrict__ w_toff, const int32_t* __restrict__ rs_score,
                                              const uint2* __restrict__ rs_sink, uint32_t i, int32_t& score, uint32_t& end)
{
    if (!want[i]) return false;
    const uint32_t j = job_idx[i];
    if (j >= pp.rescue_capacity) return false;
    score = rs_score[j];
    if (score < pp.min_mate_score) return false;
    end = w_toff[i] + rs_sink[j].x;
    return true;
}

__global__ void __launch_bounds__(256)
pair_finalize_kernel(const uint32_t n_pairs, const nvb_pair_params pp, const uint32_t* __restrict__ want, const uint32_t* __restrict__ job_idx,
                     const uint32_t* __restrict__ w_toff, const int32_t* __restrict__ rs_score, const uint2* __restrict__ rs_sink,
                     int32_t* __restrict__ pair_score, uint32_t* __restrict__ pair_flags,
                     int32_t* __restrict__ mate_score, uint32_t* __restrict__ mate_pos, uint8_t* __restrict__ mate_strand)
{
    const uint32_t p = blockIdx.x * 256 + threadIdx.x;
    if (p >= n_pairs || pair_flags[p] == NVB_PAIR_CONCORDANT) return;
    int best_a = -1; int32_t best_sum = INT_MIN, best_rs = 0; uint32_t best_pos = 0;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
        int32_t rs; uint32_t end;
        if (!usable_rescue(pp, want, job_idx, w_toff, rs_score, rs_sink, 2 * p + a, rs, end)) continue;
        const int32_t sum = mate_score[a * n_pairs + p] + rs;
        if (sum > best_sum) { best_sum = sum; best_a = a; best_rs = rs; best_pos = end; }
    }
    if (best_a < 0) return;
    const int o = 1 - best_a;
    pair_score[p] = best_sum;
    pair_flags[p] = o == 0 ? NVB_PAIR_RESCUED_MATE1 : NVB_PAIR_RESCUED_MATE2;
    mate_score[o * n_pairs + p] = best_rs;
    mate_pos[o * n_pairs + p] = best_pos;
    mate_strand[o * n_pairs + p] = (uint8_t)(1u - mate_strand[best_a * n_pairs + p]);
}

// ---------------------------------------------------------------------------------------------
// paired-end traceback (nvb_seed_extend_paired_traceback): mates that keep their single-end best take its banded traceback; a rescued
// mate takes the full-matrix traceback of the winning opposite-mate job (gotoh_full_warp_traceback_kernel from its known sink)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool pair_rescued(uint32_t flags) { return flags == NVB_PAIR_RESCUED_MATE1 || flags == NVB_PAIR_RESCUED_MATE2; }

// a rescued mate's alignment is overwritten by the rescue's: its banded traceback job is emptied (mate m of pair p = read m * n_pairs + p)
__global__ void __launch_bounds__(256)
pair_empty_rescued_jobs_kernel(const uint32_t n_pairs, const uint32_t* __restrict__ pair_flags, uint32_t* __restrict__ bp_len, uint32_t* __restrict__ bt_len)
{
    const uint32_t p = blockIdx.x * 256 + threadIdx.x;
    if (p >= n_pairs) return;
    const uint32_t f = pair_flags[p];
    if (!pair_rescued(f)) return;
    const uint32_t r = (f == NVB_PAIR_RESCUED_MATE1 ? 0u : n_pairs) + p;
    bp_len[r] = 0; bt_len[r] = 0;
}

// the winning job of every rescued pair (the job of anchor a = the mate not rescued, the one pair_finalize_kernel chose) as a traceback
// item (job index into the rescue list, rescued mate); one atomic per warp.  The rescued mate's strand goes to ba_strand (may be NULL)
__global__ void __launch_bounds__(256)
pair_rescue_items_kernel(const uint32_t n_pairs, const uint32_t* __restrict__ pair_flags, const uint32_t* __restrict__ job_idx,
                         const uint8_t* __restrict__ mate_strand, uint2* __restrict__ items, uint32_t* __restrict__ n_items, uint8_t* __restrict__ ba_strand)
{
    const uint32_t p = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31u;
    const uint32_t f = p < n_pairs ? pair_flags[p] : 0u;
    const bool rescued = pair_rescued(f);
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, rescued);
    if (!m) return;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(n_items, (uint32_t)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (!rescued) return;
    const uint32_t o = f == NVB_PAIR_RESCUED_MATE1 ? 0u : 1u, out = o * n_pairs + p;
    items[base + __popc(m & ((1u << lane) - 1u))] = make_uint2(job_idx[2u * p + (1u - o)], out);
    if (ba_strand) ba_strand[out] = mate_strand[out];
}

// ---------------------------------------------------------------------------------------------
// second-best pair and paired MAPQ (nvb_seed_extend_paired_mapq).  The candidates of a mate are those of the single-end stage (see
// pipe_second_reduce_kernel) that reach the read's min score, gathered into one segment per read, sorted by (strand, end) and merged per
// (strand, end); pair_second_kernel pairs them up (pair_combinations, pipeline_core.cuh) and adds the pair's rescues.
// ---------------------------------------------------------------------------------------------

// one thread per read: its sorted segment merged per (strand, end) into the one with the highest (score, -tie), written to m_end / m_score
// / m_tie from the segment's start; n_fw / n_merged = forward / all merged candidates
__global__ void __launch_bounds__(256)
pair_cand_merge_kernel(const uint32_t n_reads, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ cnt,
                       const unsigned long long* __restrict__ key, const uint32_t* __restrict__ val, const Scored c,
                       uint32_t* __restrict__ m_end, int32_t* __restrict__ m_score, uint32_t* __restrict__ m_tie,
                       uint32_t* __restrict__ n_fw, uint32_t* __restrict__ n_merged)
{
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= n_reads) return;
    const uint32_t b = seg[r], n = cnt[r];
    uint32_t m = 0, fw = 0; unsigned long long prev = ~0ull;
    for (uint32_t k = b; k < b + n; ++k) {
        const unsigned long long kk = key[k];
        const uint32_t j = val[k], tie = c.tie(j);
        const int32_t sc = c.score[j];
        if (kk == prev) {
            const uint32_t o = b + m - 1u;
            if (sc > m_score[o] || (sc == m_score[o] && tie < m_tie[o])) { m_score[o] = sc; m_tie[o] = tie; }
            continue;
        }
        prev = kk;
        m_end[b + m] = (uint32_t)kk; m_score[b + m] = sc; m_tie[b + m] = tie;
        ++m; if ((kk >> 32) == 0ull) ++fw;
    }
    n_fw[r] = fw; n_merged[r] = m;
}

// one thread per pair: the second-best pair (combinations of the mates' candidates plus the pair's rescues) and the MAPQ of both mates.
// UNPAIRED pairs keep the single-end MAPQ pipe_mapq_kernel wrote into mate_mapq.  se_pos: the mates' single-end best ends (a rescue's
// anchor), best_key: their tie indices
__global__ void __launch_bounds__(256)
pair_second_kernel(const uint32_t n_pairs, const nvb_pair_params pp, const nvb_mapq_params mp, const uint32_t* __restrict__ str_len,
                   const uint32_t* __restrict__ seg, const uint32_t* __restrict__ n_fw, const uint32_t* __restrict__ n_merged,
                   const uint32_t* __restrict__ m_end, const int32_t* __restrict__ m_score, const uint32_t* __restrict__ m_tie,
                   const uint32_t* __restrict__ se_pos, const uint8_t* __restrict__ se_strand, const unsigned long long* __restrict__ best_key,
                   const uint32_t* __restrict__ want, const uint32_t* __restrict__ job_idx, const uint32_t* __restrict__ w_toff,
                   const int32_t* __restrict__ rs_score, const uint2* __restrict__ rs_sink,
                   const int32_t* __restrict__ pair_score, const uint32_t* __restrict__ pair_flags,
                   const uint32_t* __restrict__ mate_pos, const uint8_t* __restrict__ mate_strand,
                   int32_t* __restrict__ second_pair_score, uint32_t* __restrict__ second_mate_pos, uint8_t* __restrict__ second_mate_strand,
                   uint8_t* __restrict__ mate_mapq)
{
    const uint32_t p = blockIdx.x * 256 + threadIdx.x;
    if (p >= n_pairs) return;
    const uint32_t r0 = p, r1 = n_pairs + p;
    const uint32_t len[2] = {str_len[2u * r0], str_len[2u * r1]};         // (both strands of a read have its length)
    PairSecond ps;
    ps.init(mate_pos[r0], mate_strand[r0], len[0], mate_pos[r1], mate_strand[r1], len[1]);
    const uint32_t flags = pair_flags[p];
    if (flags != NVB_PAIR_UNPAIRED) {
        MateCands m[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint32_t r = k ? r1 : r0, b = seg[r];
            m[k].end = m_end + b; m[k].score = m_score + b; m[k].tie = m_tie + b; m[k].n_fw = n_fw[r]; m[k].n = n_merged[r]; m[k].len = len[k];
        }
        pair_combinations(m, pp.min_frag, pp.max_frag, ps);
        // rescues: the anchor's single-end best with the rescued alignment of the other mate (tie index 0xFFFFFFFF)
        for (int a = 0; a < 2; ++a) {
            const uint32_t ra = a ? r1 : r0;
            int32_t rs; uint32_t end;
            if (!usable_rescue(pp, want, job_idx, w_toff, rs_score, rs_sink, 2u * p + a, rs, end) || rs < mp.d_min_score[len[1 - a]]) continue;
            const unsigned long long key = best_key[ra];
            ps.offer_rescue(a, best_key_score(key) + rs, se_pos[ra], se_strand[ra], best_key_index(key), end);
        }
        const uint8_t q = (uint8_t)bowtie_mapq2(pair_score[p], ps.has, ps.score, (int32_t)(len[0] + len[1]) * mp.match_bonus,
                                                mp.d_min_score[len[0]] + mp.d_min_score[len[1]], mp.match_bonus == 0);
        mate_mapq[r0] = q; mate_mapq[r1] = q;
    }
    second_pair_score[p] = ps.score;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        if (second_mate_pos) second_mate_pos[k * n_pairs + p] = ps.end[k];
        if (second_mate_strand) second_mate_strand[k * n_pairs + p] = (uint8_t)ps.strand[k];
    }
}

} // namespace nvb

using namespace nvb;

// stage boundaries of the most recent nvb_seed_extend call ON EACH DEVICE (events are recorded on the caller's stream; they
// cost no synchronisation).  [0]=start, then after: strings, seed match, slots, locate+windows, job dedup, extension, reduce.
// Events belong to the device that created them, so the set is per device, created under a mutex on first use; a host that
// drives several GPUs from one process (one compute thread per device) gets one set per GPU.  Callers that run several
// batches of one device concurrently (nvb_pipeline) pass their own events instead.
struct StageEvents { cudaEvent_t ev[8]; bool ready, valid; };
static StageEvents g_stage[NVB_MAX_DEVICES];
static std::mutex  g_stage_mutex;
static int default_stage_events(StageEvents** out)
{
    int dev = 0;
    NVB_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= NVB_MAX_DEVICES) return NVB_E_UNSUPPORTED;
    std::lock_guard<std::mutex> lock(g_stage_mutex);
    StageEvents& S = g_stage[dev];
    if (!S.ready) {
        for (int i = 0; i < 8; ++i) NVB_CUDA_TRY(cudaEventCreate(&S.ev[i]));
        S.ready = true;
    }
    *out = &S;
    return NVB_OK;
}

extern "C" int nvb_seed_extend_stage_ms(float ms[7])
{
    if (!ms) return NVB_E_INVALID;
    StageEvents* SE = nullptr;
    { const int r = default_stage_events(&SE); if (r != NVB_OK) return r; }
    if (!SE->valid) return NVB_E_INVALID;
    NVB_CUDA_TRY(cudaEventSynchronize(SE->ev[7]));
    for (int i = 0; i < 7; ++i) NVB_CUDA_TRY(cudaEventElapsedTime(&ms[i], SE->ev[i], SE->ev[i + 1]));
    return NVB_OK;
}

static int g_perfect_shortcut = 1;     // 0 = every alignment job through the DP kernels, 2 = without the one-gap check (nvb_debug_perfect_shortcut)
static const uint32_t* g_last_dp_count = nullptr;   // the last per-read call's count of jobs left to the DP (nvb_debug_dp_jobs)
static int g_seed_split = 1;           // 0 = the located seed match in one pass (nvb_debug_seed_split)
static int g_pipe_path = 0;            // 1 = always the per-hit path, anything else = automatic (nvb_debug_pipeline_path)

#define NVB_TRY(expr) do { const int _r = (expr); if (_r != NVB_OK) return _r; } while (0)
static int size_only(int r) { return r == NVB_E_TEMP_SIZE ? NVB_OK : r; }     // a temp-size query's answer: its error, if any
static int launched() { return (int)cudaGetLastError(); }                       // the launches' error, if any (cudaSuccess == NVB_OK)

// a list whose length (<= n) lives on the device: a resident grid of 256-thread CTAs striding over it (16 per SM) instead of n / 256
// mostly empty CTAs
static uint32_t resident_grid(uint32_t n) { const uint32_t grid = (n + 255) / 256, cap = sm_count() * 16u; return grid < cap ? grid : cap; }

static Jobs take_jobs(TempCarver& tc, size_t n) { return Jobs{tc.take<uint32_t>(n), tc.take<uint32_t>(n), tc.take<uint32_t>(n), tc.take<uint32_t>(n)}; }
struct JobViews { nvb_string_set pats, txts; };

// one seed + extend call as an entry point states it: inputs, per-read and per-hit outputs (the per-hit ones may be NULL) and the
// optional groups, NULL when not asked for: BA best-alignment traceback, PP / PO pairs, MP / MO MAPQ, PMO paired MAPQ, AP / AO k alignments
struct SeedExtendReq {
    const nvb_fm_index* fmi; const uint32_t* genome; const nvb_string_set* reads; uint32_t n_reads; const nvb_seed_extend_params* P; uint32_t hit_capacity;
    int32_t* best_score; uint32_t* best_pos; uint32_t* n_hits; uint32_t* hit_read; nvb_uint2* hit_window; int32_t* hit_score; nvb_uint2* hit_sink;
    const nvb_best_alignment_out* BA; const nvb_pair_params* PP; const nvb_pair_out* PO;
    const nvb_mapq_params* MP; const nvb_mapq_out* MO; const nvb_pair_mapq_out* PMO;
    const nvb_all_params* AP; const nvb_all_out* AO;
};

// one call: its request, the path it takes, its temp buffers (NULL in the size query and where the path does not use them), its stages
struct PipeCall : SeedExtendReq {
    PipeGeom g; cudaStream_t s; FmIndex f; StrSet rd;
    uint32_t nq;
    bool dedup, per_read, eligible;                                         // eligible: the exact shortcut applies (gapless_job_shortcut)
    bool seed_split;                                                        // the located seed match in two passes (match_seeds)
    nvb_mapq_out se_mo;                                                     // paired MAPQ: the single-end stage's outputs (MO = &se_mo)
    StageEvents* SE;
    uint32_t *str_words, *str_len; uint8_t* str_quals;                      // [fw, rc] strings
    uint2* ranges; uint32_t *sizes, *excl, *counts, *seed_todo, *seed_todo_n;   // counts: [0] hits kept, [1] hits found, [2] alignment jobs
    char* rj_tiles; size_t rj_tile_bytes;                                   // per-read path: tile states of the hit-slot look-back
    uint32_t *j_string, *j_first;                                           // per-read path: string and first hit of every job
    uint32_t *leader, *flag, *job_idx;                                      // per-hit path: job de-duplication
    Jobs jobs; int32_t* job_score; uint2* job_sink;                         // the distinct jobs (dedup_jobs)
    Jobs dp; uint32_t *dp_job, *dp_count; int32_t* dp_score; uint2* dp_sink;   // the jobs the exact shortcut leaves to the DP
    uint32_t* hit_string; Jobs hits; int32_t* h_score; uint2* h_sink;       // per-hit path: every hit
    unsigned long long* best_key; uint8_t* rb_strand;                       // best alignment of every read, its strand
    char *scan_tmp, *gotoh_tmp; size_t scan_bytes, gotoh_bytes;
    Jobs best; int32_t* b_score; uint2 *b_sink, *b_source; char* tb_tmp; size_t tb_bytes;      // best-alignment traceback
    uint32_t *pw_want, *pw_idx, *pw_pstr, *pw_toff, *pw_tlen, *pcounts;     // paired: two opposite-mate job slots per pair
    Jobs rescue; int32_t* rs_score; uint2* rs_sink; char *pscan_tmp, *full_tmp; size_t pscan_bytes, full_bytes;
    uint2* rt_items; uint32_t* rt_count; char* rt_pool; size_t rt_pool_bytes;   // paired traceback (PP and BA): rescued mates, warp slot pool
    unsigned long long* second_key;                                        // second-best alignment of every read (MO)
    uint32_t *cs_cnt, *cs_seg, *cs_val[2]; unsigned long long* cs_key[2];  // candidate segments (PMO or AO), their scan and sort
    char *cs_scan_tmp, *cs_sort_tmp; size_t cs_scan_bytes, cs_sort_bytes;
    uint32_t *pc_fw, *pc_n, *pc_end, *pc_tie, *se_pos; int32_t* pc_score;   // paired MAPQ (PMO): merged candidates per read
    uint32_t *al_slice_n, n_slices; Jobs al_jobs;                           // nvb_seed_extend_all: traceback slices, jobs

    int stage(int i) const { return (int)cudaEventRecord(SE->ev[i], s); }    // boundary i of nvb_seed_extend_stage_ms

    // a job list's read strings vs genome windows (<= txt_len); in the size queries any non-null words pointer does
    JobViews job_views(const Jobs& j, uint32_t txt_len) const
    {
        //        d_words                                      bits    big_endian  d_offsets  d_lengths  stride  length
        return {{str_words ? str_words : (const uint32_t*)16,  g.bits, 1u,         j.p_off,   j.p_len,   0u,     rd.length},
                {genome,                                       2u,     1u,         j.t_off,   j.t_len,   0u,     txt_len}};
    }

    // banded extension of the first *d_n (<= hit_capacity) jobs of a list
    int score_jobs(const Jobs& j, const uint32_t* d_n, int32_t* score, uint2* sink) const
    {
        const JobViews v = job_views(j, rd.length + g.band);
        size_t bytes = gotoh_bytes;
        return nvb_banded_gotoh_score_indirect(g.band, P->type, &P->scheme, &v.pats, str_quals, &v.txts, d_n, hit_capacity,
                                               score, (nvb_uint2*)sink, gotoh_tmp, &bytes, s);
    }

    // every temp buffer in one pass: with d_temp == NULL (the size query) the pointers stay NULL and only `need` counts
    int carve(void* d_temp, size_t& need)
    {
        const uint32_t cap = hit_capacity, n_reads = g.n_reads;
        const JobViews sv = job_views(Jobs{}, rd.length + g.band);
        NVB_TRY(size_only(nvb_banded_gotoh_score(g.band, P->type, &P->scheme, &sv.pats, nullptr, &sv.txts, cap, nullptr, nullptr, nullptr,
                                                 &gotoh_bytes, s)));
        TempCarver tc(d_temp);
        str_words = tc.take<uint32_t>((size_t)g.n_strings * (g.stride / (32u / g.bits)) + 4);
        str_len   = tc.take<uint32_t>(g.n_strings);
        str_quals = P->d_read_quals ? tc.take<uint8_t>((size_t)g.n_strings * g.stride + 16) : nullptr;
        ranges = tc.take<uint2>(nq);
        if (!per_read) { sizes = tc.take<uint32_t>(nq); excl = tc.take<uint32_t>(nq); }
        if (seed_split) seed_todo = tc.take<uint32_t>((size_t)nq + (SEED_TODO_LISTS + 1u) * SEED_BLOCK * SEED_ITER);   // lists' capacity, see pipe_seed_match_kernel
        counts = tc.take<uint32_t>(4); seed_todo_n = tc.take<uint32_t>(SEED_TODO_LISTS * SEED_TODO_PITCH);
        if (per_read) {
            NVB_CUDA_TRY(RjTileState::AllocationSize((int)((n_reads + RJ_BLOCK - 1u) / RJ_BLOCK), rj_tile_bytes));
            rj_tiles = tc.take<char>(rj_tile_bytes);
        }
        if (per_read) { j_string = tc.take<uint32_t>(cap); j_first = tc.take<uint32_t>(cap); }
        else if (dedup) { leader = tc.take<uint32_t>(cap); flag = tc.take<uint32_t>(cap); job_idx = tc.take<uint32_t>(cap); }
        if (dedup) { jobs = take_jobs(tc, cap); job_score = tc.take<int32_t>(cap); job_sink = tc.take<uint2>(cap); }
        if (per_read) {                                              // the jobs the exact shortcut leaves to the DP (all of them when it is off)
            dp = take_jobs(tc, cap); dp_job = tc.take<uint32_t>(cap); dp_score = tc.take<int32_t>(cap); dp_sink = tc.take<uint2>(cap);
            dp_count = tc.take<uint32_t>(4);
        }
        if (!per_read) { hit_string = tc.take<uint32_t>(cap); hits = take_jobs(tc, cap); }
        h_score = hit_score ? hit_score : (per_read ? nullptr : tc.take<int32_t>(cap));
        h_sink  = hit_sink ? (uint2*)hit_sink : (per_read ? nullptr : tc.take<uint2>(cap));
        best_key = tc.take<unsigned long long>(n_reads); rb_strand = tc.take<uint8_t>((size_t)n_reads + 16);
        scan_bytes = 0;
        if (!per_read) NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, sizes, excl, (int)nq, s));
        if (dedup && !per_read && cap) {
            size_t scan2_bytes = 0;
            NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan2_bytes, flag, job_idx, (int)cap, s));
            if (scan2_bytes > scan_bytes) scan_bytes = scan2_bytes;
        }
        scan_tmp  = tc.take<char>(scan_bytes);
        gotoh_tmp = tc.take<char>(gotoh_bytes);
        if (BA || AO) {                                              // nvb_seed_extend_all: one slice of n_reads alignments at a time
            if (BA) best = take_jobs(tc, n_reads);
            b_score = tc.take<int32_t>(n_reads); b_sink = tc.take<uint2>(n_reads); b_source = tc.take<uint2>(n_reads);
            NVB_TRY(size_only(nvb_banded_gotoh_traceback(g.band, P->type, &P->scheme, &sv.pats, nullptr, &sv.txts, n_reads, nullptr, nullptr,
                                                         nullptr, nullptr, BA ? BA->max_ops : AO->alignment.max_ops, nullptr, nullptr, &tb_bytes, s)));
            tb_tmp = tc.take<char>(tb_bytes);
        }
        if (PP) {
            const uint32_t rcap = PP->rescue_capacity;
            pw_want = tc.take<uint32_t>(n_reads); pw_idx = tc.take<uint32_t>(n_reads); pw_pstr = tc.take<uint32_t>(n_reads);
            pw_toff = tc.take<uint32_t>(n_reads); pw_tlen = tc.take<uint32_t>(n_reads); pcounts = tc.take<uint32_t>(4);
            rescue = take_jobs(tc, rcap); rs_score = tc.take<int32_t>(rcap); rs_sink = tc.take<uint2>(rcap);
            NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, pscan_bytes, pw_want, pw_idx, (int)n_reads, s));
            pscan_tmp = tc.take<char>(pscan_bytes);
            const JobViews v = job_views(Jobs{}, PP->max_frag);
            NVB_TRY(size_only(nvb_gotoh_score_indirect(P->type, &P->scheme, &v.pats, nullptr, &v.txts, (const uint32_t*)16, rcap, nullptr, nullptr,
                                                       nullptr, &full_bytes, s)));
            full_tmp = tc.take<char>(full_bytes);
            if (BA) {
                NVB_TRY(full_warp_traceback(P->type, rd.length, PP->max_frag, nullptr, &rt_pool_bytes, s));
                rt_items = tc.take<uint2>((size_t)n_reads / 2u + 1u); rt_count = tc.take<uint32_t>(4); rt_pool = tc.take<char>(rt_pool_bytes);
            }
        }
        if (MO) second_key = tc.take<unsigned long long>(n_reads);
        if (PMO || AO) {
            cs_cnt = tc.take<uint32_t>((size_t)n_reads + 1); cs_seg = tc.take<uint32_t>((size_t)n_reads + 1);
            for (int k = 0; k < 2; ++k) { cs_key[k] = tc.take<unsigned long long>(cap); cs_val[k] = tc.take<uint32_t>(cap); }
            NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, cs_scan_bytes, cs_cnt, cs_seg, (int)n_reads + 1, s));
            cs_scan_tmp = tc.take<char>(cs_scan_bytes);
            cs_sort_bytes = 0;
            if (cap) NVB_CUDA_TRY(cub::DeviceSegmentedSort::SortPairs(nullptr, cs_sort_bytes, cs_key[0], cs_key[1], cs_val[0], cs_val[1], (int)cap,
                                                                     (int)n_reads, cs_seg, cs_seg + 1, s));
            cs_sort_tmp = tc.take<char>(cs_sort_bytes);
        }
        if (PMO) {
            if (!PMO->d_mate_second_score) se_mo.d_second_score = tc.take<int32_t>(n_reads);
            pc_fw = tc.take<uint32_t>(n_reads); pc_n = tc.take<uint32_t>(n_reads); se_pos = tc.take<uint32_t>(n_reads);
            pc_end = tc.take<uint32_t>(cap); pc_score = tc.take<int32_t>(cap); pc_tie = tc.take<uint32_t>(cap);
        }
        if (AO) {
            const uint32_t acap = AP->capacity;
            n_slices = n_reads ? (uint32_t)(((uint64_t)acap + n_reads - 1u) / n_reads) : 0u;
            al_jobs = take_jobs(tc, acap); al_slice_n = tc.take<uint32_t>((size_t)n_slices + 1);
        }
        need = tc.total();
        return NVB_OK;
    }

    // 1. [fw, rc] strings and their base qualities
    int make_strings() const
    {
        const uint32_t grid = (uint32_t)(((uint64_t)g.n_strings * (g.stride / (32u / g.bits)) + 255) / 256);     // one thread per word
        if (g.bits == 2 && rd.big_endian) pipe_make_strings_2bit_be_kernel<<<grid, 256, 0, s>>>(rd, g, str_words, str_len);
        else if (g.bits == 2)             pipe_make_strings_kernel<2><<<grid, 256, 0, s>>>(rd, g, str_words, str_len);
        else                              pipe_make_strings_kernel<4><<<grid, 256, 0, s>>>(rd, g, str_words, str_len);
        NVB_LAUNCH_CHECK();
        if (str_quals) pipe_make_quals_kernel<<<(uint32_t)(((uint64_t)g.n_strings * g.stride + 255) / 256), 256, 0, s>>>(rd, g, P->d_read_quals, str_quals);
        return launched();
    }

    // 2. seed ranges.  Per-read path + full suffix array: single-row ranges are located inside the match kernel; with a k-mer table in
    // two passes (seed_split), seeds on k-mers with >= 3 occurrences finished by a second kernel.  The per-read path stores no sizes
    int match_seeds() const
    {
        const uint32_t grid = (nq + SEED_BLOCK - 1) / SEED_BLOCK;
        const uint32_t* loc_genome = (per_read && f.sa_shift == 0u) ? genome : nullptr;
        if (seed_split) {
            NVB_CUDA_TRY(cudaMemsetAsync(seed_todo_n, 0, SEED_TODO_LISTS * SEED_TODO_PITCH * sizeof(uint32_t), s));
            const uint32_t grid1 = (grid + SEED_ITER - 1u) / SEED_ITER;
            if (g.bits == 2) pipe_seed_match_kernel<2, true><<<grid1, SEED_BLOCK, 0, s>>>(f, g, str_words, str_len, loc_genome, ranges, sizes, seed_todo, seed_todo_n);
            else             pipe_seed_match_kernel<4, true><<<grid1, SEED_BLOCK, 0, s>>>(f, g, str_words, str_len, loc_genome, ranges, sizes, seed_todo, seed_todo_n);
            NVB_LAUNCH_CHECK();
            const uint32_t wgrid = (sm_count() * 16u + SEED_TODO_LISTS - 1u) / SEED_TODO_LISTS * SEED_TODO_LISTS;   // 16 resident CTAs per SM (H100: 2112), whole lists
            if (g.bits == 2) pipe_seed_match_wide_kernel<2><<<wgrid, SEED_BLOCK, 0, s>>>(f, g, str_words, loc_genome, ranges, sizes, seed_todo, seed_todo_n, grid1);
            else             pipe_seed_match_wide_kernel<4><<<wgrid, SEED_BLOCK, 0, s>>>(f, g, str_words, loc_genome, ranges, sizes, seed_todo, seed_todo_n, grid1);
        } else {
            if (g.bits == 2) pipe_seed_match_kernel<2, false><<<grid, SEED_BLOCK, 0, s>>>(f, g, str_words, str_len, loc_genome, ranges, sizes, nullptr, nullptr);
            else             pipe_seed_match_kernel<4, false><<<grid, SEED_BLOCK, 0, s>>>(f, g, str_words, str_len, loc_genome, ranges, sizes, nullptr, nullptr);
        }
        return launched();
    }

    // 4'-6'. per-read path: hit slots, locate, window, distinct jobs, exact shortcut and the claimed best per read in one kernel (stage 4),
    // the DP over the jobs left to it and their scatter into the best per read (6), the DP winners' results (7)
    int extend_per_read() const
    {
        const nvb_gotoh_scheme& SC = P->scheme;
        const uint32_t cap = hit_capacity, n_tiles = (g.n_reads + RJ_BLOCK - 1u) / RJ_BLOCK;
        RjTileState tiles;
        NVB_CUDA_TRY(tiles.Init((int)n_tiles, rj_tiles, rj_tile_bytes));
        pipe_resolve_init_kernel<<<(n_tiles + 255u) / 256u, 256, 0, s>>>(tiles, n_tiles, counts, dp_count);
        NVB_LAUNCH_CHECK();
        const int shortcut = eligible ? g_perfect_shortcut : 0;
        const int32_t max_gap_open = SC.pattern_gap_open > SC.text_gap_open ? SC.pattern_gap_open : SC.text_gap_open;
        pipe_resolve_reads_kernel<<<n_tiles, RJ_BLOCK, 0, s>>>(f, g, ranges, str_len, cap, tiles, n_tiles, counts, shortcut, SC.match,
                SC.mismatch, max_gap_open, str_words, genome, j_string, j_first, jobs, job_score, job_sink, dp, dp_job, dp_count,
                best_key, best_score, best_pos, rb_strand);
        NVB_LAUNCH_CHECK();
        g_last_dp_count = dp_count;
        NVB_TRY(stage(4)); NVB_TRY(stage(5));
        const uint32_t jgrid = resident_grid(cap);
        if (cap) {
            NVB_TRY(score_jobs(dp, dp_count, dp_score, dp_sink));
            pipe_scatter_dp_kernel<<<jgrid, 256, 0, s>>>(g, dp_count, dp_job, dp_score, dp_sink, j_string, j_first, job_score, job_sink, best_key);
            NVB_LAUNCH_CHECK();
        }
        NVB_TRY(stage(6));
        if (cap) {
            pipe_finalize_dp_kernel<<<jgrid, 256, 0, s>>>(g, dp_count, dp_job, dp_score, dp_sink, dp.t_off, j_string, j_first, best_key,
                                                          best_score, best_pos, rb_strand);
            NVB_LAUNCH_CHECK();
        }
        return launched();
    }

    // 4-6. per-hit path: locate + window per hit (4), collapse identical (string, window) jobs (5), extension (6), best hit per read
    int extend_per_hit() const
    {
        const uint32_t cap = hit_capacity, hgrid = (cap + 255) / 256;
        if (cap) {
            pipe_expand_hits_kernel<<<(nq + 255) / 256, 256, 0, s>>>(f, g, ranges, sizes, excl, str_len, counts,
                                                                     hit_string, hits.p_off, hits.p_len, hits.t_off, hits.t_len);
            NVB_LAUNCH_CHECK();
        }
        NVB_TRY(stage(4));
        if (dedup && cap) {
            pipe_find_leaders_kernel<<<hgrid, 256, 0, s>>>(counts, hit_string, hits.t_off, hits.t_len, leader, flag);
            NVB_LAUNCH_CHECK();
            // the scan runs over the whole capacity; job_idx[h] depends only on flag[0..h), so the (unwritten) entries
            // past counts[0] cannot influence any index that is read back
            size_t bytes = scan_bytes;
            NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, bytes, flag, job_idx, (int)cap, s));
            pipe_job_count_kernel<<<1, 32, 0, s>>>(job_idx, flag, counts);
            NVB_LAUNCH_CHECK();
            pipe_compact_jobs_kernel<<<hgrid, 256, 0, s>>>(counts, flag, job_idx, hits.p_off, hits.p_len, hits.t_off, hits.t_len,
                                                           jobs.p_off, jobs.p_len, jobs.t_off, jobs.t_len);
            NVB_LAUNCH_CHECK();
        }
        NVB_TRY(stage(5));
        NVB_CUDA_TRY(cudaMemsetAsync(best_key, 0, sizeof(unsigned long long) * g.n_reads, s));
        if (cap && dedup) {
            NVB_TRY(score_jobs(jobs, counts + 2, job_score, job_sink));
            pipe_scatter_scores_kernel<<<hgrid, 256, 0, s>>>(g, counts, leader, job_idx, job_score, job_sink, hit_string, h_score, h_sink, best_key);
            NVB_LAUNCH_CHECK();
        } else if (cap)
            NVB_TRY(score_jobs(hits, counts, h_score, h_sink));
        NVB_TRY(stage(6));
        // with job de-duplication the best-per-read reduction already happened in the scatter kernel
        if (cap && !dedup) {
            pipe_reduce_kernel<<<hgrid, 256, 0, s>>>(g, counts, hit_string, h_score, h_sink, best_key);
            NVB_LAUNCH_CHECK();
        }
        pipe_finalize_kernel<<<(g.n_reads + 255) / 256, 256, 0, s>>>(g, best_key, hits.t_off, h_sink, hit_string, best_score, best_pos, rb_strand);
        return launched();
    }

    // best-alignment traceback: the best hit of every read as a job, its banded traceback, the alignment's begin in the genome
    // (per-read path: the best job of every read from the distinct jobs; paired: after the rescue, whose rescued mates get empty jobs)
    int best_traceback() const
    {
        const uint32_t rgrid = (g.n_reads + 255) / 256;
        if (per_read) {
            pipe_empty_jobs_kernel<<<rgrid, 256, 0, s>>>(g.n_reads, best.p_off, best.p_len, best.t_off, best.t_len, BA->d_strand);
            NVB_LAUNCH_CHECK();
            const uint32_t jgrid = resident_grid(hit_capacity);
            if (jgrid) {
                pipe_winner_kernel<<<jgrid, 256, 0, s>>>(g, scored(), best_key, best, nullptr, BA->d_strand);
                NVB_LAUNCH_CHECK();
            }
        } else {
            pipe_best_jobs_kernel<<<rgrid, 256, 0, s>>>(g, best_key, hit_string, hits.p_off, hits.p_len, hits.t_off, hits.t_len,
                                                        best.p_off, best.p_len, best.t_off, best.t_len, BA->d_strand);
            NVB_LAUNCH_CHECK();
        }
        if (PP) {
            const uint32_t n_pairs = g.n_reads / 2u;
            pair_empty_rescued_jobs_kernel<<<(n_pairs + 255) / 256, 256, 0, s>>>(n_pairs, PO->d_pair_flags, best.p_len, best.t_len);
            NVB_LAUNCH_CHECK();
        }
        return trace_jobs(best, nullptr, g.n_reads, *BA, 0, best_key);
    }

    // banded traceback of the first n jobs of a list (d_n != NULL: *d_n <= n of them) into alignments [off, off + n) of A, in the
    // best-alignment traceback's temp buffers; best_key != NULL: job r is read r's best (see traceback_begin_kernel)
    int trace_jobs(const Jobs& j, const uint32_t* d_n, uint32_t n, const nvb_best_alignment_out& A, size_t off, const unsigned long long* key) const
    {
        const JobViews v = job_views(j, rd.length + g.band);
        size_t bytes = tb_bytes;
        NVB_TRY(banded_traceback(g.band, P->type, &P->scheme, &v.pats, str_quals, &v.txts, d_n, n, b_score, (nvb_uint2*)b_sink,
                                 (nvb_uint2*)b_source, A.d_ops + off * A.max_ops, A.max_ops, A.d_n_ops + off, tb_tmp, &bytes, s));
        traceback_begin_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_n, n, key, j.t_off, b_source, A.d_n_ops + off, (uint2*)A.d_begin + off);
        return launched();
    }

    // the alignments the extension scored: the per-read path's distinct jobs, the per-hit path's kept hits
    Scored scored() const
    {
        return per_read ? Scored{counts + 2, j_string, j_first, jobs, job_score, job_sink} : Scored{counts, hit_string, nullptr, hits, h_score, h_sink};
    }

    // second-best distinct alignment and MAPQ of every read: one more pass over the scored alignments, after the best alignment is known
    int second_best() const
    {
        NVB_CUDA_TRY(cudaMemsetAsync(second_key, 0, sizeof(unsigned long long) * g.n_reads, s));
        if (hit_capacity) {
            const uint32_t grid = resident_grid(hit_capacity);
            pipe_second_reduce_kernel<<<grid, 256, 0, s>>>(g, scored(), str_len, best_pos, rb_strand, MP->d_min_score, second_key);
            NVB_LAUNCH_CHECK();
            if (MO->d_second_pos || MO->d_second_strand) {
                pipe_winner_kernel<<<grid, 256, 0, s>>>(g, scored(), second_key, Jobs{}, MO->d_second_pos, MO->d_second_strand);
                NVB_LAUNCH_CHECK();
            }
        }
        pipe_mapq_kernel<<<(g.n_reads + 255) / 256, 256, 0, s>>>(g, *MP, str_len, best_score, second_key, MO->d_second_score, MO->d_second_pos,
                                                                MO->d_second_strand, MO->d_mapq);
        return launched();
    }

    // every read's candidates (those second_best() sees that reach its min score) in a segment of their own, [cs_seg[r], + cs_cnt[r]),
    // sorted by (strand, end) or, by_best, in rank order (descending make_best_key): keys in cs_key[1], candidates in cs_val[1];
    // cs_cnt[n_reads] = 0
    int cand_segments(bool by_best) const
    {
        const uint32_t cap = hit_capacity, n_reads = g.n_reads;
        NVB_CUDA_TRY(cudaMemsetAsync(cs_cnt, 0, sizeof(uint32_t) * ((size_t)n_reads + 1), s));
        if (cap) {
            const uint32_t grid = resident_grid(cap);
            cand_scatter_kernel<<<grid, 256, 0, s>>>(g, scored(), str_len, MP->d_min_score, nullptr, cs_cnt, nullptr, nullptr, by_best);
            NVB_LAUNCH_CHECK();
            size_t bytes = cs_scan_bytes;
            NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cs_scan_tmp, bytes, cs_cnt, cs_seg, (int)n_reads + 1, s));
            NVB_CUDA_TRY(cudaMemsetAsync(cs_cnt, 0, sizeof(uint32_t) * n_reads, s));
            cand_scatter_kernel<<<grid, 256, 0, s>>>(g, scored(), str_len, MP->d_min_score, cs_seg, cs_cnt, cs_key[0], cs_val[0], by_best);
            NVB_LAUNCH_CHECK();
            bytes = cs_sort_bytes;
            NVB_CUDA_TRY(cub::DeviceSegmentedSort::SortPairs(cs_sort_tmp, bytes, cs_key[0], cs_key[1], cs_val[0], cs_val[1], (int)cap, (int)n_reads,
                                                             cs_seg, cs_seg + 1, s));
        } else
            NVB_CUDA_TRY(cudaMemsetAsync(cs_seg, 0, sizeof(uint32_t) * ((size_t)n_reads + 1), s));
        return NVB_OK;
    }

    // paired MAPQ, before the rescue overwrites the mate arrays: the candidate segments merged per (strand, end); the single-end best ends
    // (rescue anchors)
    int pair_candidates() const
    {
        NVB_CUDA_TRY(cudaMemcpyAsync(se_pos, best_pos, sizeof(uint32_t) * g.n_reads, cudaMemcpyDeviceToDevice, s));
        NVB_TRY(cand_segments(false));
        pair_cand_merge_kernel<<<(g.n_reads + 255) / 256, 256, 0, s>>>(g.n_reads, cs_seg, cs_cnt, cs_key[1], cs_val[1], scored(), pc_end, pc_score,
                                                                        pc_tie, pc_fw, pc_n);
        return launched();
    }

    // up to k distinct alignments of every read (after second_best: the same candidates), each traced; no host round trip
    int all_alignments() const
    {
        const uint32_t n_reads = g.n_reads, acap = AP->capacity, rgrid = (n_reads + 255) / 256;
        const nvb_all_out& O = *AO;
        NVB_TRY(cand_segments(true));
        // cs_cnt[n_reads] stays 0: the scan's extra element makes d_first[n_reads] the total
        all_select_kernel<<<rgrid, 256, 0, s>>>(g, scored(), str_len, cs_seg, cs_key[1], cs_val[1], AP->max_per_read, cs_cnt);
        NVB_LAUNCH_CHECK();
        size_t bytes = cs_scan_bytes;
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cs_scan_tmp, bytes, cs_cnt, O.d_first, (int)n_reads + 1, s));
        all_count_kernel<<<(n_slices + 256) / 256, 256, 0, s>>>(n_reads, O.d_first, acap, n_slices, O.d_count, al_slice_n);
        NVB_LAUNCH_CHECK();
        if (!acap) return launched();
        all_emit_kernel<<<rgrid, 256, 0, s>>>(g, scored(), O.d_first, cs_seg, cs_val[1], acap, O.d_read, O.d_score, O.d_pos, O.alignment.d_strand,
                                              al_jobs);
        NVB_LAUNCH_CHECK();
        // slice t: alignments [t * n_reads, + n) traced like the best alignments of nvb_seed_extend_traceback (its direction matrices, sized
        // for n_reads); the count of each slice lives on the device, a slice past the stored alignments launches only empty CTAs
        for (uint32_t t = 0; t < n_slices; ++t) {
            const size_t b = (size_t)t * n_reads;
            const Jobs j{al_jobs.p_off + b, al_jobs.p_len + b, al_jobs.t_off + b, al_jobs.t_len + b};
            NVB_TRY(trace_jobs(j, al_slice_n + t, (uint32_t)(acap - b < n_reads ? acap - b : n_reads), O.alignment, b, nullptr));
        }
        return launched();
    }

    // second-best pair and MAPQ of every pair, after the rescue: the pairs' final flags and mates are P*
    int pair_second() const
    {
        const uint32_t n_pairs = g.n_reads / 2u;
        pair_second_kernel<<<(n_pairs + 255) / 256, 256, 0, s>>>(n_pairs, *PP, *MP, str_len, cs_seg, pc_fw, pc_n, pc_end, pc_score, pc_tie,
                                                                  se_pos, rb_strand, best_key, pw_want, pw_idx, pw_toff, rs_score, rs_sink,
                                                                  PO->d_pair_score, PO->d_pair_flags, PO->d_mate_pos, PO->d_mate_strand,
                                                                  PMO->d_second_pair_score, PMO->d_second_mate_pos, PMO->d_second_mate_strand,
                                                                  PMO->d_mate_mapq);
        return launched();
    }

    // paired-end rescue: non-concordant pairs get opposite-mate jobs (scan-compacted) for the full-matrix DP; the best rescue wins
    int paired_rescue() const
    {
        const uint32_t n_reads = g.n_reads, n_pairs = n_reads / 2u, cap = PP->rescue_capacity;
        const uint32_t pgrid = (n_pairs + 255) / 256, sgrid = (n_reads + 255) / 256;
        pair_classify_kernel<<<pgrid, 256, 0, s>>>(g, n_pairs, *PP, best_score, best_pos, rb_strand, str_len, pw_want, pw_pstr, pw_toff, pw_tlen,
                                                    PO->d_pair_score, PO->d_pair_flags, PO->d_mate_score, PO->d_mate_pos, PO->d_mate_strand);
        NVB_LAUNCH_CHECK();
        size_t bytes = pscan_bytes;
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(pscan_tmp, bytes, pw_want, pw_idx, (int)n_reads, s));
        pipe_count_kernel<<<1, 32, 0, s>>>(pw_idx, pw_want, n_reads, cap, pcounts);      // [0] jobs run (<= capacity), [1] jobs wanted
        NVB_LAUNCH_CHECK();
        if (cap) {
            pair_compact_kernel<<<sgrid, 256, 0, s>>>(g, n_reads, cap, pw_want, pw_idx, pw_pstr, pw_toff, pw_tlen, str_len,
                                                      rescue.p_off, rescue.p_len, rescue.t_off, rescue.t_len);
            NVB_LAUNCH_CHECK();
            const JobViews v = job_views(rescue, PP->max_frag);
            size_t fb = full_bytes;
            NVB_TRY(nvb_gotoh_score_indirect(P->type, &P->scheme, &v.pats, str_quals, &v.txts, pcounts, cap, rs_score, (nvb_uint2*)rs_sink, full_tmp, &fb, s));
        }
        pair_finalize_kernel<<<pgrid, 256, 0, s>>>(n_pairs, *PP, pw_want, pw_idx, pw_toff, rs_score, rs_sink, PO->d_pair_score, PO->d_pair_flags,
                                                    PO->d_mate_score, PO->d_mate_pos, PO->d_mate_strand);
        NVB_LAUNCH_CHECK();
        if (PO->d_n_rescue) NVB_CUDA_TRY(cudaMemcpyAsync(PO->d_n_rescue, pcounts, 2 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
        return NVB_OK;
    }

    // paired traceback of the rescued mates (after best_traceback, whose outputs they overwrite): the winning opposite-mate job of every
    // rescued pair, traced from the rescue score pass's sink on its window; begin = (window begin + source.x, source.y)
    int rescue_traceback() const
    {
        const uint32_t n_pairs = g.n_reads / 2u;
        NVB_CUDA_TRY(cudaMemsetAsync(rt_count, 0, sizeof(uint32_t), s));
        pair_rescue_items_kernel<<<(n_pairs + 255) / 256, 256, 0, s>>>(n_pairs, PO->d_pair_flags, pw_idx, PO->d_mate_strand, rt_items, rt_count,
                                                                       BA->d_strand);
        NVB_LAUNCH_CHECK();
        const JobViews v = job_views(rescue, PP->max_frag);
        FullTbArgs a;
        a.S = make_scheme(&P->scheme); a.pat = make_strset(&v.pats); a.txt = make_strset(&v.txts); a.quals = str_quals;
        a.score = rs_score; a.sink = rs_sink; a.items = rt_items; a.n_items = rt_count;
        a.o.ops = BA->d_ops; a.o.n_ops = BA->d_n_ops; a.o.source = (uint2*)BA->d_begin; a.o.max_ops = BA->max_ops; a.o.absolute = 1u;
        a.pool = rt_pool;
        size_t bytes = rt_pool_bytes;
        return full_warp_traceback(P->type, rd.length, PP->max_frag, &a, &bytes, s);
    }
};

static int seed_extend_impl(const SeedExtendReq& R, void* d_temp, size_t* temp_bytes, void* stream)
{
    // The entry points check only what cannot be seen here: that the structs they require are there, and the pair count before
    // 2 * n_pairs is formed.  The order below decides which code a call with several faults gets: the paired traceback's read length
    // limit comes after the outputs and MAPQ inputs and before everything else.
    if (!R.reads || !temp_bytes) return NVB_E_INVALID;
    if (R.BA && (!R.BA->d_ops || !R.BA->d_n_ops || !R.BA->d_begin || R.BA->max_ops == 0)) return NVB_E_INVALID;
    if ((R.MP == nullptr) != (R.MO == nullptr && R.PMO == nullptr)) return NVB_E_INVALID;
    if (R.MP && (!R.MP->d_min_score || R.MP->max_read_len < R.reads->length)) return NVB_E_INVALID;   // the min-score table must cover every read length
    if (R.MO && (!R.MO->d_second_score || !R.MO->d_mapq)) return NVB_E_INVALID;
    if (R.PMO && (!R.PMO->d_second_pair_score || !R.PMO->d_mate_mapq)) return NVB_E_INVALID;
    if (R.PP && R.BA && R.reads->length > FULL_TB_MAX_M) return NVB_E_UNSUPPORTED;                 // nvBowtie's MAXIMUM_READ_LENGTH
    if (R.AO && R.reads->length > FULL_TB_MAX_M) return NVB_E_UNSUPPORTED;
    const nvb_seed_extend_params* P = R.P;
    if (R.PP) {
        if (!R.PO->d_pair_score || !R.PO->d_pair_flags || !R.PO->d_mate_score || !R.PO->d_mate_pos || !R.PO->d_mate_strand) return NVB_E_INVALID;
        if (!P || !P->both_strands || (R.n_reads & 1u) || R.PP->max_frag == 0 || R.PP->min_frag > R.PP->max_frag) return NVB_E_INVALID;
    }
    if (!valid_fmindex(R.fmi) || !R.fmi->d_ssa || !R.genome || !valid_strset(R.reads) || !P) return NVB_E_INVALID;
    if (R.reads->bits == 8) return NVB_E_UNSUPPORTED;
    if (P->seed_len == 0 || P->seed_interval == 0 || P->max_seed_hits == 0) return NVB_E_INVALID;
    if (R.n_reads && (!R.best_score || !R.best_pos)) return NVB_E_INVALID;
    const uint32_t max_len = R.reads->length;               // maximum read length (== length for fixed-length sets)
    if (max_len < P->seed_len) return NVB_E_INVALID;

    PipeCall c{R};                                          // the request; everything else starts zeroed
    PipeGeom& g = c.g;
    g.n_reads = R.n_reads; g.strands = P->both_strands ? 2u : 1u; g.n_strings = R.n_reads * g.strands;
    g.bits = R.reads->bits;
    const uint32_t spw = 32u / g.bits;
    g.stride = (max_len + spw - 1u) / spw * spw;
    g.seeds_per_string = (max_len - P->seed_len) / P->seed_interval + 1u;
    g.seed_len = P->seed_len; g.seed_interval = P->seed_interval; g.band = P->band_len;
    g.max_seed_hits = P->max_seed_hits; g.genome_len = R.fmi->length;
    if ((uint64_t)g.n_strings * g.stride > 0xFFFFFFFFull) return NVB_E_UNSUPPORTED;
    const uint64_t nq64 = (uint64_t)g.n_strings * g.seeds_per_string;
    if (nq64 > 0x7FFFFFFFull) return NVB_E_UNSUPPORTED;
    // hit slots are a uint32 exclusive sum of the clamped range sizes: the worst case must fit
    if (nq64 * (uint64_t)P->max_seed_hits > 0xFFFFFFFFull) return NVB_E_UNSUPPORTED;

    const cudaStream_t s = c.s = as_stream(stream);
    c.f = make_fmindex(R.fmi); c.rd = make_strset(R.reads); c.nq = (uint32_t)nq64;
    if (R.PMO) {                               // the single-end second best and MAPQ of every mate (mate_mapq: overwritten for paired pairs)
        c.se_mo.d_second_score = R.PMO->d_mate_second_score; c.se_mo.d_mapq = R.PMO->d_mate_mapq;
        c.MO = &c.se_mo;
    }
    c.dedup = P->dedup_jobs != 0;
    // per-read path: nobody asked for per-hit outputs, so no per-hit array needs to exist (the traceback takes the best of the distinct jobs)
    c.per_read = c.dedup && g_pipe_path != 1 && !R.hit_read && !R.hit_window && !R.hit_score && !R.hit_sink;
    const nvb_gotoh_scheme& SC = P->scheme;
    c.eligible = c.per_read && P->type == NVB_LOCAL && g.bits == 2 && P->band_len <= 32 && !SC.d_qual_table && SC.match > 0 && SC.mismatch < 0 &&
                 SC.pattern_gap_open < 0 && SC.pattern_gap_ext <= 0 && SC.text_gap_open < 0 && SC.text_gap_ext <= 0;
    c.seed_split = c.per_read && c.f.sa_shift == 0u && c.f.ktab_k && g.seed_len > c.f.ktab_k && g_seed_split;
    size_t need = 0;
    NVB_TRY(c.carve(d_temp, need));
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (R.n_reads == 0) {
        if (R.AO) {
            NVB_CUDA_TRY(cudaMemsetAsync(R.AO->d_first, 0, sizeof(uint32_t), s));
            NVB_CUDA_TRY(cudaMemsetAsync(R.AO->d_count, 0, 2 * sizeof(uint32_t), s));
        }
        return NVB_OK;
    }

    NVB_TRY(default_stage_events(&c.SE));
    NVB_TRY(c.stage(0));
    NVB_TRY(c.make_strings()); NVB_TRY(c.stage(1));
    NVB_TRY(c.match_seeds());  NVB_TRY(c.stage(2));
    // 3. per-hit path: hit slots, the exclusive sum of the clamped range sizes (the per-read path takes them inside its stage 4)
    if (!c.per_read) {
        size_t scan_bytes = c.scan_bytes;
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c.scan_tmp, scan_bytes, c.sizes, c.excl, (int)c.nq, s));
        pipe_count_kernel<<<1, 32, 0, s>>>(c.excl, c.sizes, c.nq, R.hit_capacity, c.counts);
        NVB_LAUNCH_CHECK();
    }
    NVB_TRY(c.stage(3));
    NVB_TRY(c.per_read ? c.extend_per_read() : c.extend_per_hit());       // records stages 4 to 6
    if (R.hit_capacity && (R.hit_read || R.hit_window)) {
        pipe_export_hits_kernel<<<(R.hit_capacity + 255) / 256, 256, 0, s>>>(g, c.counts, c.hit_string, c.hits.t_off, c.hits.t_len, R.hit_read,
                                                                             (uint2*)R.hit_window);
        NVB_LAUNCH_CHECK();
    }
    if (R.BA && !R.PP) NVB_TRY(c.best_traceback());
    if (c.MO) NVB_TRY(c.second_best());
    if (R.AO) NVB_TRY(c.all_alignments());
    if (R.PMO) NVB_TRY(c.pair_candidates());
    if (R.PP) NVB_TRY(c.paired_rescue());
    if (R.BA && R.PP) { NVB_TRY(c.best_traceback()); NVB_TRY(c.rescue_traceback()); }
    if (R.PMO) NVB_TRY(c.pair_second());
    if (!c.dedup) NVB_CUDA_TRY(cudaMemcpyAsync(c.counts + 2, c.counts, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    if (R.n_hits) NVB_CUDA_TRY(cudaMemcpyAsync(R.n_hits, c.counts, 3 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    NVB_TRY(c.stage(7));
    c.SE->valid = true;
    return NVB_OK;
}

extern "C" void nvb_debug_pipeline_path(int path) { g_pipe_path = path; }
extern "C" void nvb_debug_seed_split(int on) { g_seed_split = on; }
extern "C" void nvb_debug_perfect_shortcut(int on) { g_perfect_shortcut = on; }
extern "C" int nvb_debug_dp_jobs(uint32_t* n)
{
    if (!n || !g_last_dp_count) return NVB_E_INVALID;
    NVB_CUDA_TRY(cudaDeviceSynchronize());
    NVB_CUDA_TRY(cudaMemcpy(n, g_last_dp_count, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return NVB_OK;
}

extern "C" int nvb_seed_extend(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    void* d_temp, size_t* temp_bytes, void* stream)
{
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = n_reads; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = d_best_score; R.best_pos = d_best_pos; R.n_hits = d_n_hits; R.hit_read = d_hit_read; R.hit_window = d_hit_window;
    R.hit_score = d_hit_score; R.hit_sink = d_hit_sink;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_traceback(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!best_alignment) return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = n_reads; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = d_best_score; R.best_pos = d_best_pos; R.n_hits = d_n_hits; R.hit_read = d_hit_read; R.hit_window = d_hit_window;
    R.hit_score = d_hit_score; R.hit_sink = d_hit_sink; R.BA = best_alignment;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_paired(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!pair_params || !out || n_pairs > 0x3FFFFFFFu) return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = 2u * n_pairs; R.P = P; R.hit_capacity = hit_capacity;
    // the per-read best (score, end) of the single-end stage lands in the mate arrays first and is then refined per pair
    R.best_score = out->d_mate_score; R.best_pos = out->d_mate_pos; R.n_hits = d_n_hits; R.PP = pair_params; R.PO = out;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_mapq(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    const nvb_mapq_params* mapq, const nvb_mapq_out* mapq_out,
                    void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!mapq || !mapq_out) return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = n_reads; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = d_best_score; R.best_pos = d_best_pos; R.n_hits = d_n_hits; R.hit_read = d_hit_read; R.hit_window = d_hit_window;
    R.hit_score = d_hit_score; R.hit_sink = d_hit_sink; R.BA = best_alignment; R.MP = mapq; R.MO = mapq_out;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_all(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    const nvb_mapq_params* mapq, const nvb_mapq_out* mapq_out,
                    const nvb_all_params* all_params, const nvb_all_out* all_out,
                    void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!mapq || !mapq_out || !all_params || !all_out || best_alignment) return NVB_E_INVALID;
    const nvb_all_out& O = *all_out;
    const nvb_best_alignment_out& A = O.alignment;
    if (!O.d_first || !O.d_read || !O.d_score || !O.d_pos || !O.d_count || !A.d_ops || !A.d_n_ops || !A.d_begin || !A.d_strand || A.max_ops == 0)
        return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = n_reads; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = d_best_score; R.best_pos = d_best_pos; R.n_hits = d_n_hits; R.hit_read = d_hit_read; R.hit_window = d_hit_window;
    R.hit_score = d_hit_score; R.hit_sink = d_hit_sink; R.MP = mapq; R.MO = mapq_out; R.AP = all_params; R.AO = all_out;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_paired_mapq(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    const nvb_mapq_params* mapq, const nvb_pair_mapq_out* mapq_out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!pair_params || !out || !mapq || !mapq_out || n_pairs > 0x3FFFFFFFu) return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = 2u * n_pairs; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = out->d_mate_score; R.best_pos = out->d_mate_pos; R.n_hits = d_n_hits; R.PP = pair_params; R.PO = out; R.MP = mapq; R.PMO = mapq_out;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_seed_extend_paired_traceback(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* P, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    const nvb_best_alignment_out* mate_alignment,
                    const nvb_mapq_params* mapq, const nvb_pair_mapq_out* mapq_out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!pair_params || !out || !mate_alignment || n_pairs > 0x3FFFFFFFu) return NVB_E_INVALID;
    SeedExtendReq R = {};
    R.fmi = fmi; R.genome = d_genome; R.reads = reads; R.n_reads = 2u * n_pairs; R.P = P; R.hit_capacity = hit_capacity;
    R.best_score = out->d_mate_score; R.best_pos = out->d_mate_pos; R.n_hits = d_n_hits; R.PP = pair_params; R.PO = out;
    R.BA = mate_alignment; R.MP = mapq; R.PMO = mapq_out;
    return seed_extend_impl(R, d_temp, temp_bytes, stream);
}

extern "C" int nvb_debug_mapq_eval(const int32_t* d_best, const uint8_t* d_has_second, const int32_t* d_second, const uint32_t* d_len,
                                   const int32_t* d_match_bonus, const int32_t* d_min_score, uint32_t n, uint8_t* d_mapq, void* stream)
{
    if (!n) return NVB_OK;
    if (!d_best || !d_has_second || !d_second || !d_len || !d_match_bonus || !d_min_score || !d_mapq) return NVB_E_INVALID;
    debug_mapq_eval_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(d_best, d_has_second, d_second, d_len, d_match_bonus, d_min_score, n, d_mapq);
    return launched();
}
