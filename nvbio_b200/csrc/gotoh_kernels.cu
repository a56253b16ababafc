// gotoh_kernels.cu -- HP-B: batched banded Gotoh scoring kernels and their C ABI.
//
//   gotoh_pair_kernel<B,TYPE>     two alignments per thread in s16x2 halves (DPX), text selectors staged
//                                 in shared memory (one conflict-free u16 column per thread); pairs that
//                                 violate the packed path's preconditions are appended to a todo list
//   gotoh_generic_kernel<B,TYPE>  one alignment per thread, int32, every symbol width / quality table;
//                                 runs over the whole batch or over the todo list
//
// The path is bound by integer issue rate, not memory: ~0.1 KB moved per 4,650 cell updates (B=31, M=150).
#include "gotoh_core.cuh"
#include <atomic>
#include "../../include/nvbio_b200_debug.h"
#include "gotoh_full_core.cuh"
#include "pipeline_core.cuh"

namespace nvb {

static int g_traceback_fast = 1;        // nvb_debug_traceback_fast(0): every alignment through the full (direction-matrix) traceback
static int g_pair_extra_smem = 0;       // nvb_debug_pair_extra_smem: bytes of unused dynamic shared memory added to every pair-kernel CTA (occupancy experiments)
static int g_pair_rows2 = 1;            // nvb_debug_pair_rows2(0): one row per loop iteration in the pair kernels
static bool g_pair_fmt_ok = true;       // nvb_debug_pair_format(0) forces the run-time-format kernel (tests compare the two)

constexpr int PAIR_BLOCKDIM    = 128;
constexpr int GENERIC_BLOCKDIM = 128;

struct GotohBatch {
    StrSet   pat, txt;
    const uint8_t* quals;
    const uint32_t* d_n;       // optional device-side count
    uint32_t n_max;
    int32_t* score;
    uint2*   sink;
};

__device__ __forceinline__ uint32_t batch_count(const GotohBatch& b) {
    if (!b.d_n) return b.n_max;
    const uint32_t n = *b.d_n;
    return n < b.n_max ? n : b.n_max;
}

template <int B, int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_generic_kernel(const GotohScheme S, const GotohBatch b, const uint32_t* __restrict__ todo, const uint32_t* __restrict__ todo_count)
{
    const uint32_t n = todo ? *todo_count : batch_count(b);
    for (uint32_t t = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x; t < n; t += gridDim.x * GENERIC_BLOCKDIM) {
        const uint32_t a = todo ? todo[t] : t;
        const SinkResult r = gotoh_generic<B, TYPE>(S,
            b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), str_len(b.pat, a), b.quals,
            b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a));
        b.score[a] = r.score;
        b.sink[a]  = make_uint2(r.x, r.y);
    }
}

// Best2Sink variant of the int32 kernel: out6[a] = (score1, sink1.x, sink1.y, score2, sink2.x, sink2.y)
template <int B, int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_best2_kernel(const GotohScheme S, const GotohBatch b, uint32_t distinct_dist, int32_t* __restrict__ out6)
{
    const uint32_t n = batch_count(b);
    const uint32_t a = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x;
    if (a >= n) return;
    Best2 b2; b2.init(distinct_dist);
    gotoh_generic_impl<B, TYPE, false>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), str_len(b.pat, a), b.quals,
                                       b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a), nullptr, &b2);
    int32_t* o = out6 + 6 * (size_t)a;
    o[0] = b2.s1; o[1] = (int32_t)b2.x1; o[2] = (int32_t)b2.y1; o[3] = b2.s2; o[4] = (int32_t)b2.x2; o[5] = (int32_t)b2.y2;
}
template <int B, int TYPE>
static int launch_best2(const GotohScheme& S, const GotohBatch& b, uint32_t distinct_dist, int32_t* out6, cudaStream_t s)
{
    gotoh_best2_kernel<B, TYPE><<<(b.n_max + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM, GENERIC_BLOCKDIM, 0, s>>>(S, b, distinct_dist, out6);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

// a word of sixteen 2-bit symbols with their order reversed (little-endian <-> big-endian symbol order)
__device__ __forceinline__ uint32_t swap_2bit_order(uint32_t x) {
    const uint32_t r = __brev(x);
    return ((r >> 1) & 0x55555555u) | ((r & 0x55555555u) << 1);
}

// one pair of alignments (2 pair, 2 pair + 1) of gotoh_pair_kernel, n = the batch size; my_sel = the thread's selector column
template <int B, int TYPE, int PFMT, bool ROWS2>
__device__ __forceinline__ void gotoh_pair_job(const GotohScheme& S, const GotohBatch& b, const uint32_t sel_rows, uint32_t* __restrict__ todo,
                                               uint32_t* __restrict__ todo_count, const uint32_t pair, const uint32_t n, uint16_t* my_sel,
                                               const uint32_t* prof_tab)
{
    const uint32_t a0 = 2u * pair;
    const bool has1 = (a0 + 1u < n);
    const uint32_t a1 = has1 ? a0 + 1u : a0;          // an odd tail computes the same alignment in both halves

    const uint32_t M0 = str_len(b.pat, a0), M1 = str_len(b.pat, a1);
    const uint32_t N0 = str_len(b.txt, a0), N1 = str_len(b.txt, a1);
    const uint32_t Mmax = M0 > M1 ? M0 : M1;
    const uint32_t L = Mmax + (uint32_t)B - 1u;       // text columns touched

    const bool ok = (M0 >= 1u) && (M1 >= 1u) && (N0 >= M0 + (uint32_t)B - 1u) && (N1 >= M1 + (uint32_t)B - 1u) &&
                    (L <= sel_rows) && (TYPE == NVB_LOCAL || M0 == M1);
    if (!ok) {
        const uint32_t cnt = has1 ? 2u : 1u;
        const uint32_t slot = atomicAdd(todo_count, cnt);
        todo[slot] = a0;
        if (has1) todo[slot + 1u] = a1;
        return;
    }

    // stage the PRMT selectors of this thread's two text windows (own shared-memory column: no barrier needed).
    // Word-wise: the 16 symbols starting at any offset are a funnel shift of two consecutive words, and the loads
    // of successive words are independent, so they overlap instead of forming a chain of dependent round trips.
    {
        const uint32_t t0 = str_off(b.txt, a0), t1 = str_off(b.txt, a1);
        const uint32_t* __restrict__ w = b.txt.words;
        const bool be = b.txt.big_endian != 0;
        const uint32_t w0 = t0 >> 4, w1 = t1 >> 4;                         // first stream word of each window
        const uint32_t sh0 = 2u * (t0 & 15u), sh1 = 2u * (t1 & 15u);
        const uint32_t last0 = (t0 + N0 - 1u) >> 4, last1 = (t1 + N1 - 1u) >> 4;   // last word holding a window symbol
        const uint32_t nw = (L + 15u) >> 4;
        // the window words are fetched eight (+1) per alignment at a time, all loads of a batch independent of each other: a
        // thread pays two or three DRAM round trips for its two windows instead of one per word (the windows sit at random
        // genome positions, and at 16 warps per SM nobody else hides that latency)
        // (the shared array is sized for whole words of 16 columns, so no per-column bound checks: symbols past a window's end
        // are masked to 0 per word, columns past L are written and never read)
        for (uint32_t kb = 0; kb < nw; kb += 8u) {
            uint32_t a0[9], a1[9];
#pragma unroll
            for (uint32_t q = 0; q < 9u; ++q) {
                // never touch a word beyond the window's last one
                a0[q] = (w0 + kb + q <= last0) ? w[w0 + kb + q] : 0u;
                a1[q] = (w1 + kb + q <= last1) ? w[w1 + kb + q] : 0u;
            }
#pragma unroll
            for (uint32_t q = 0; q < 8u; ++q) {
                const uint32_t k = kb + q;
                if (k < nw) {
                    uint32_t c0, c1;
                    if (be) {
                        c0 = sh0 ? ((a0[q] << sh0) | (a0[q + 1] >> (32u - sh0))) : a0[q];
                        c1 = sh1 ? ((a1[q] << sh1) | (a1[q + 1] >> (32u - sh1))) : a1[q];
                    } else {
                        c0 = sh0 ? ((a0[q] >> sh0) | (a0[q + 1] << (32u - sh0))) : a0[q];
                        c1 = sh1 ? ((a1[q] >> sh1) | (a1[q + 1] << (32u - sh1))) : a1[q];
                    }
                    const uint32_t first = k << 4;
                    // symbols of this word inside the window: v0, v1 in [0, 16]; the rest read as symbol 0
                    const uint32_t v0 = N0 > first ? (N0 - first < 16u ? N0 - first : 16u) : 0u;
                    const uint32_t v1 = N1 > first ? (N1 - first < 16u ? N1 - first : 16u) : 0u;
                    const uint32_t m0 = v0 >= 16u ? 0xFFFFFFFFu : (be ? ~(0xFFFFFFFFu >> (2u * v0)) : ((1u << (2u * v0)) - 1u));
                    const uint32_t m1 = v1 >= 16u ? 0xFFFFFFFFu : (be ? ~(0xFFFFFFFFu >> (2u * v1)) : ((1u << (2u * v1)) - 1u));
                    c0 &= m0; c1 &= m1;
                    if (!be) { c0 = swap_2bit_order(c0); c1 = swap_2bit_order(c1); }        // first symbol in the top bits from here on
                    // four columns at a time: one byte of each window side by side, then per column a shift, a mask and an IMAD
                    //   x = g0 | g1 << 8;  pair_selector(g0, g1) = 0xC480 + x * 0x11
#pragma unroll
                    for (uint32_t by = 0; by < 4u; ++by) {
                        const uint32_t W = prmt(c0, c1, (3u - by) | ((7u - by) << 4) | 0x3200u);      // byte `by` (from the top) of c0 | of c1 << 8
#pragma unroll
                        for (uint32_t m = 0; m < 4u; ++m) {
                            const uint32_t x = (W >> (6u - 2u * m)) & 0x0303u;
                            my_sel[(first + 4u * by + m) * PAIR_BLOCKDIM] = (uint16_t)(x * 0x11u + 0xC480u);
                        }
                    }
                }
            }
        }
    }

    SinkResult r0, r1;
    gotoh_pair<B, TYPE, PFMT, ROWS2>(S, b.pat.words, b.pat.bits, b.pat.big_endian,
                        str_off(b.pat, a0), M0, str_off(b.pat, a1), M1, N0, N1,
                        my_sel, PAIR_BLOCKDIM, r0, r1, b.quals, prof_tab);
    b.score[a0] = r0.score; b.sink[a0] = make_uint2(r0.x, r0.y);
    if (has1) { b.score[a1] = r1.score; b.sink[a1] = make_uint2(r1.x, r1.y); }
}

// ROWS2: two pattern rows in flight per thread (gotoh_pair)
// TICKET (only with a device-side count, b.d_n): a resident grid whose warps claim 32 pairs at a time from the ticket todo_count[1]
// (zeroed with todo_count[0]), so the launch costs what the batch holds and not what its capacity could.  Sized from the capacity
// (one pair per thread, the exact-count path), most of a pipeline batch's CTAs would start only to find no work: each still reserves
// its selector shared memory, fills prof_tab and reads *d_n before it leaves.
template <int B, int TYPE, int PFMT, bool ROWS2, bool TICKET>
__global__ void __launch_bounds__(PAIR_BLOCKDIM, 4)
gotoh_pair_kernel(const GotohScheme S, const GotohBatch b, uint32_t sel_rows, uint32_t* __restrict__ todo, uint32_t* __restrict__ todo_count)
{
    extern __shared__ uint16_t sel_smem[];            // [sel_rows rounded up to 16][PAIR_BLOCKDIM]
    // substitution profile of every possible pattern symbol (constant schemes): one LDS per row instead of building it
    __shared__ uint32_t prof_tab[256];
    for (uint32_t q = threadIdx.x; q < 256u; q += PAIR_BLOCKDIM) prof_tab[q] = sub_profile(q, S.match - S.pgo, S.mismatch - S.pgo);
    __syncthreads();
    const uint32_t n = batch_count(b);
    const uint32_t n_pairs = (n + 1u) / 2u;
    uint16_t* my_sel = sel_smem + threadIdx.x;
    if (!TICKET) {
        // one pair per thread (a grid-stride loop over a resident grid measured 5% slower: 108 vs 118 registers cost
        // more than the empty CTAs of a device-side count save)
        const uint32_t pair = blockIdx.x * PAIR_BLOCKDIM + threadIdx.x;
        if (pair >= n_pairs) return;
        gotoh_pair_job<B, TYPE, PFMT, ROWS2>(S, b, sel_rows, todo, todo_count, pair, n, my_sel, prof_tab);
    } else {
        const uint32_t lane = threadIdx.x & 31u;
        for (;;) {
            uint32_t first = 0;
            if (lane == 0u) first = atomicAdd(todo_count + 1, 32u);
            first = __shfl_sync(0xFFFFFFFFu, first, 0);
            if (first >= n_pairs) return;
            if (first + lane < n_pairs) gotoh_pair_job<B, TYPE, PFMT, ROWS2>(S, b, sel_rows, todo, todo_count, first + lane, n, my_sel, prof_tab);
        }
    }
}

// full-matrix Gotoh: one alignment per thread, 32-column register stripes, boundary column in HBM scratch laid out
// [text row][alignment] so that a warp's accesses to one row are contiguous
template <int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_full_kernel(const GotohScheme S, const GotohBatch b, int2* __restrict__ col)
{
    const uint32_t n = batch_count(b);
    const uint32_t a = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x;
    if (a >= n) return;
    const SinkResult r = gotoh_full<TYPE>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), str_len(b.pat, a),
                                          b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a),
                                          col + a, (size_t)b.n_max, b.quals);
    b.score[a] = r.score;
    b.sink[a]  = make_uint2(r.x, r.y);
}

// windowed scoring: one alignment per thread, rows [wb, min(we, M)); checkpoints, BestSinks and alive flags live in HBM between passes
struct WindowArgs { uint32_t wb, we; const int32_t* min_score; short2* ckpt; uint8_t* alive; };

template <int B, int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_window_kernel(const GotohScheme S, const GotohBatch b, const WindowArgs w)
{
    const uint32_t n = batch_count(b);
    const uint32_t a = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x;
    if (a >= n) return;
    SinkResult r;
    if (w.wb == 0) { r.score = NVB_SINK_MIN; r.x = r.y = 0xFFFFFFFFu; b.score[a] = r.score; b.sink[a] = make_uint2(r.x, r.y); w.alive[a] = 1; }
    else { if (!w.alive[a]) return; r.score = b.score[a]; const uint2 k = b.sink[a]; r.x = k.x; r.y = k.y; }
    const uint32_t M = str_len(b.pat, a);
    if (w.wb >= M) return;
    const bool ok = gotoh_window<B, TYPE>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), M, b.quals,
                                          b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a),
                                          w.wb, w.we < M ? w.we : M, w.min_score ? w.min_score[a] : INT_MIN, w.ckpt + (size_t)a * B, r);
    b.score[a] = r.score; b.sink[a] = make_uint2(r.x, r.y);
    w.alive[a] = ok ? 1 : 0;
}

template <int B, int TYPE>
static int launch_window(const GotohScheme& S, const GotohBatch& b, const WindowArgs& w, cudaStream_t s)
{
    const uint32_t grid = (b.n_max + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM;
    gotoh_window_kernel<B, TYPE><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, w);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

struct TracebackOut {
    uint2* source; uint8_t* ops; uint32_t* n_ops; uint32_t max_ops; uint32_t* dirs; uint32_t dir_rows;
};

// full-matrix traceback: one alignment per thread; the DP writes one uint4 of direction nibbles per (text row, 32-column
// stripe) to the alignment's slot, the same thread then walks it back from the sink
template <int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_full_traceback_kernel(const GotohScheme S, const GotohBatch b, int2* __restrict__ col, const TracebackOut o, const uint32_t dir_row_words)
{
    const uint32_t n = batch_count(b);
    const uint32_t a = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x;
    if (a >= n) return;
    uint32_t* dirs = o.dirs + (size_t)a * o.dir_rows * dir_row_words;
    const uint32_t M = str_len(b.pat, a), N = str_len(b.txt, a);
    SinkResult r; r.score = NVB_SINK_MIN; r.x = r.y = 0xFFFFFFFFu;
    if (N <= o.dir_rows && (M + 31u) / 32u * 4u <= dir_row_words)
        r = gotoh_full_impl<TYPE, true>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), M,
                                        b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), N, col + a, (size_t)b.n_max, dirs, dir_row_words, b.quals);
    b.score[a] = r.score;
    b.sink[a]  = make_uint2(r.x, r.y);
    uint32_t sx = 0xFFFFFFFFu, sy = 0xFFFFFFFFu, cnt = 0;
    if (r.x != 0xFFFFFFFFu && r.y != 0xFFFFFFFFu)
        cnt = gotoh_full_walk<TYPE>(dirs, dir_row_words, r, o.ops + (size_t)a * o.max_ops, o.max_ops, sx, sy);
    o.source[a] = make_uint2(sx, sy);
    o.n_ops[a]  = cnt;
}

// full-matrix Gotoh, packed: one PAIR of alignments per thread (a, a+1); pairs that break a precondition of the packed
// path go to the todo list and are scored by gotoh_full_todo_kernel (int32)
// QUAL: quality-dependent substitution scores (S.qtab + b.quals): per-column profiles in shared memory instead of selectors
template <int TYPE, int MINB, bool QUAL = false>
__global__ void __launch_bounds__(PAIR_BLOCKDIM, MINB)
gotoh_full_pair_kernel(const GotohScheme S, const GotohBatch b, uint2* __restrict__ col, uint32_t* __restrict__ todo, uint32_t* __restrict__ todo_count)
{
    const uint32_t n = batch_count(b);
    const uint32_t n_pairs = (n + 1u) >> 1;
    const uint32_t p = blockIdx.x * PAIR_BLOCKDIM + threadIdx.x;
    // substitution profile of every possible text symbol: one LDS per row instead of building it
    __shared__ uint32_t prof_tab[256];
    for (uint32_t g = threadIdx.x; g < 256u; g += PAIR_BLOCKDIM) prof_tab[g] = sub_profile(g, S.match - S.pgo, S.mismatch - S.pgo);
    __syncthreads();
    if (p >= n_pairs) return;
    const uint32_t a0 = 2u * p, a1 = a0 + 1u;
    const bool has1 = a1 < n;
    const uint32_t M0 = str_len(b.pat, a0), N0 = str_len(b.txt, a0);
    const uint32_t M1 = has1 ? str_len(b.pat, a1) : M0, N1 = has1 ? str_len(b.txt, a1) : N0;
    bool ok = (M0 == M1) && (N0 == N1) && M0 >= 1u && N0 >= 1u;
    SinkResult r0, r1;
    __shared__ uint16_t sel[QUAL ? 1 : FULL_W * PAIR_BLOCKDIM];
    __shared__ uint32_t colp[QUAL ? 2 * FULL_W * PAIR_BLOCKDIM : 1];
    if (ok) ok = gotoh_full_pair<TYPE, QUAL>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a0), str_off(b.pat, has1 ? a1 : a0), M0,
                                       b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a0), str_off(b.txt, has1 ? a1 : a0), N0,
                                       col + p, (size_t)((b.n_max + 1u) >> 1), QUAL ? sel : sel + threadIdx.x, PAIR_BLOCKDIM, r0, r1, prof_tab,
                                       QUAL ? colp + threadIdx.x : colp, b.quals);
    if (ok) {
        b.score[a0] = r0.score; b.sink[a0] = make_uint2(r0.x, r0.y);
        if (has1) { b.score[a1] = r1.score; b.sink[a1] = make_uint2(r1.x, r1.y); }
    } else {
        const uint32_t cnt = has1 ? 2u : 1u;
        const uint32_t slot = atomicAdd(todo_count, cnt);
        todo[slot] = a0;
        if (has1) todo[slot + 1u] = a1;
    }
}

// full-matrix Gotoh for SMALL batches: one WARP per pair of alignments.  Lane l owns pattern columns [l*W, l*W + W); at step t
// it computes text row t - l of its columns (a wavefront over the lanes), receiving the left boundary (H, E) and the row's
// substitution profile from lane l-1 by shuffle -- no boundary column in memory.  The row profiles are produced 32 rows at a
// time (lane k builds the profile of row t0 + k) and fetched by a second shuffle.  LOCAL: every lane tracks the best key
// (H << 4) | (stripe-in-lane << 3) | (column & 7) of its cells with the row kept beside it (an 8-aligned stripe boundary can
// fall inside a lane's columns: W <= 8 means at most one); the (H, stripe, row, column) maxima of the lanes are then
// max-reduced, which is the reference's report order.  Same admission rules and todo-list fallback as the pair kernel.
constexpr int WARP_BLOCKDIM = 128;

template <int TYPE, int W>
__global__ void __launch_bounds__(WARP_BLOCKDIM)
gotoh_full_warp_kernel(const GotohScheme S, const GotohBatch b, uint32_t* __restrict__ todo, uint32_t* __restrict__ todo_count)
{
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    const uint32_t n = batch_count(b);
    const uint32_t n_pairs = (n + 1u) >> 1;
    const uint32_t p = (blockIdx.x * WARP_BLOCKDIM + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (p >= n_pairs) return;                                          // whole warps leave together
    const uint32_t a0 = 2u * p, a1 = a0 + 1u;
    const bool has1 = a1 < n;
    const uint32_t M = str_len(b.pat, a0), N = str_len(b.txt, a0);
    const uint32_t M1 = has1 ? str_len(b.pat, a1) : M, N1 = has1 ? str_len(b.txt, a1) : N;
    const uint32_t po0 = str_off(b.pat, a0), po1 = str_off(b.pat, has1 ? a1 : a0);
    const uint32_t to0 = str_off(b.txt, a0), to1 = str_off(b.txt, has1 ? a1 : a0);
    bool ok = (M == M1) && (N == N1) && M >= 1u && N >= 1u && M <= 32u * (uint32_t)W;

    const int32_t Go = S.pgo, Ge = S.pge;
    const uint32_t Go2 = pack16(Go, Go), Ge2 = pack16(Ge, Ge);
    int32_t INF = SHRT_MIN - (Go < Ge ? Go : Ge);
    if (INF + Ge < -32768) INF = -32768 - Ge;
    const int32_t c_eq = S.match - Go, c_ne = S.mismatch - Go;
    const int32_t beta = -Go;
    const uint32_t beta2 = pack16(beta, beta);
    const uint32_t GoX = (uint32_t)(Go * 65537);
    const uint32_t INFx = (TYPE == NVB_LOCAL) ? pack16(INF + beta, INF + beta) : pack16(INF, INF);

    const uint32_t c0 = lane * (uint32_t)W;                            // columns c0 + 1 .. c0 + W (1-based)
    const uint32_t L = (M + (uint32_t)W - 1u) / (uint32_t)W;           // lanes that own a column
    // selectors of the lane's columns, key constants of the LOCAL tracker
    uint32_t sel[W], kmul[W], kadd[W];
    {
        uint32_t bad = 0u;
#pragma unroll
        for (int k = 0; k < W; ++k) {
            const uint32_t c = c0 + (uint32_t)k;                       // 0-based column
            uint32_t q0 = 0u, q1 = 0u;
            if (ok && c < M) { q0 = sym_at_rt(b.pat.words, b.pat.bits, b.pat.big_endian, po0 + c); q1 = sym_at_rt(b.pat.words, b.pat.bits, b.pat.big_endian, po1 + c); }
            bad |= (q0 | q1) >> 2;
            sel[k] = pair_selector(q0 & 3u, q1 & 3u);
            const uint32_t sb = (c >> 3) - (c0 >> 3);                  // 0 or 1: which 8-column stripe of this lane
            const uint32_t ka = (sb << 3) | (c & 7u);
            kmul[k] = (c < M) ? 16u : 0u;
            kadd[k] = (c < M) ? (ka | (ka << 16)) : 0u;
        }
        ok = ok && !__any_sync(FULL, bad != 0u);
    }
    if (!ok) {
        if (lane == 0u) {
            const uint32_t cnt = has1 ? 2u : 1u;
            const uint32_t slot = atomicAdd(todo_count, cnt);
            todo[slot] = a0;
            if (has1) todo[slot + 1u] = a1;
        }
        return;
    }

    // previous-row state of the lane's columns: V = H (LOCAL) or H + Go; F biased like the pair kernel
    uint32_t V[W + 1], F[W + 1];
#pragma unroll
    for (int k = 0; k <= W; ++k) {
        int32_t h = 0;
        if (TYPE != NVB_LOCAL) h = ((c0 + k > 0) ? Go + Ge * (int32_t)(c0 + k - 1) : 0) + Go;
        V[k] = pack16(h, h);
        F[k] = INFx;
    }
    uint32_t prevVl = V[0];                                            // diagonal input of the next row
    uint32_t outV = 0u, outE = 0u, curP0 = 0u, curP1 = 0u, myP0 = 0u, myP1 = 0u;
    int32_t bk0 = -1, bk1 = -1; uint32_t br0 = 0u, br1 = 0u;           // LOCAL: best key / row per half
    int32_t ss0 = INT_MIN, ss1 = INT_MIN; uint32_t sx0 = 0u, sx1 = 0u; // SEMI_GLOBAL: best score / row per half (owner lane)
    const uint32_t km = (M - 1u) % (uint32_t)W + 1u;                   // column M is V[km] of lane L - 1
    const uint32_t steps = N + L - 1u;
    for (uint32_t t = 0; t < steps; ++t) {
        if ((t & 31u) == 0u) {                                         // profiles of text rows t .. t + 31, one per lane
            const uint32_t rr = t + lane;
            uint32_t g0 = 255u, g1 = 255u;
            if (rr < N) { g0 = sym_at_rt(b.txt.words, b.txt.bits, b.txt.big_endian, to0 + rr); g1 = sym_at_rt(b.txt.words, b.txt.bits, b.txt.big_endian, to1 + rr); }
            myP0 = sub_profile(g0, c_eq, c_ne); myP1 = sub_profile(g1, c_eq, c_ne);
        }
        const uint32_t rowP0 = __shfl_sync(FULL, myP0, t & 31u), rowP1 = __shfl_sync(FULL, myP1, t & 31u);
        uint32_t inV = __shfl_up_sync(FULL, outV, 1), inE = __shfl_up_sync(FULL, outE, 1);
        uint32_t inP0 = __shfl_up_sync(FULL, curP0, 1), inP1 = __shfl_up_sync(FULL, curP1, 1);
        if (lane == 0u) {
            const int32_t hl = (TYPE == NVB_GLOBAL) ? S.tgo + S.tge * (int32_t)t + Go : ((TYPE == NVB_LOCAL) ? 0 : Go);
            inV = pack16(hl, hl);
            inE = (TYPE == NVB_LOCAL) ? beta2 : INFx;
            inP0 = rowP0; inP1 = rowP1;
        }
        const uint32_t r = t - lane;                                   // wraps for t < lane: then r >= N
        if (r < N && lane < L) {
            uint32_t E = inE, Vd = prevVl, Vleft = inV;
            prevVl = inV;
            uint32_t rowkey = 0u;
#pragma unroll
            for (int k = 1; k <= W; ++k) {
                const uint32_t s = prmt(inP0, inP1, sel[k - 1]);
                F[k] = NVB_VIADDMAX(F[k], Ge2, V[k]);
                E    = NVB_VIADDMAX(E, Ge2, Vleft);
                const uint32_t old = V[k];
                if (TYPE == NVB_LOCAL) {
                    const uint32_t hb = NVB_VIMAX3(NVB_VIADDMAX(Vd, s, F[k]), E, beta2);
                    V[k] = hb * S.one + GoX;
                    rowkey = NVB_VIMAX_U(rowkey, V[k] * kmul[k - 1] + kadd[k - 1]);
                } else {
                    V[k] = NVB_VIADD(NVB_VIMAX(NVB_VIADDMAX(Vd, s, F[k]), E), Go2);
                }
                Vleft = V[k];
                Vd = old;
            }
            outV = V[W]; outE = E; curP0 = inP0; curP1 = inP1;
            if (TYPE == NVB_LOCAL) {
                const int32_t k0 = (int32_t)(rowkey & 0xFFFFu), k1 = (int32_t)(rowkey >> 16);
                if ((k0 >> 3) >= (bk0 >> 3)) { bk0 = k0; br0 = r; }
                if ((k1 >> 3) >= (bk1 >> 3)) { bk1 = k1; br1 = r; }
            }
            if (TYPE == NVB_SEMI_GLOBAL && lane == L - 1u) {
                uint32_t vM = V[1];
#pragma unroll
                for (int k = 2; k <= W; ++k) if ((uint32_t)k == km) vM = V[k];
                const int32_t h0 = half_lo(vM) - Go, h1 = half_hi(vM) - Go;
                if (ss0 <= h0) { ss0 = h0; sx0 = r + 1u; }
                if (ss1 <= h1) { ss1 = h1; sx1 = r + 1u; }
            }
        }
    }
    // results
    SinkResult r0, r1;
    if (TYPE == NVB_LOCAL) {
        // (H, global 8-column stripe, row, column & 7) as one 64-bit key per half, max over the lanes
        unsigned long long K0 = 0ull, K1 = 0ull;
        if (lane < L) {
            K0 = ((unsigned long long)(uint32_t)(bk0 >> 4) << 32) | ((unsigned long long)((c0 >> 3) + (((uint32_t)bk0 >> 3) & 1u)) << 24) | ((unsigned long long)br0 << 3) | ((uint32_t)bk0 & 7u);
            K1 = ((unsigned long long)(uint32_t)(bk1 >> 4) << 32) | ((unsigned long long)((c0 >> 3) + (((uint32_t)bk1 >> 3) & 1u)) << 24) | ((unsigned long long)br1 << 3) | ((uint32_t)bk1 & 7u);
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            const unsigned long long o0 = __shfl_xor_sync(FULL, K0, d), o1 = __shfl_xor_sync(FULL, K1, d);
            K0 = o0 > K0 ? o0 : K0; K1 = o1 > K1 ? o1 : K1;
        }
        r0.score = (int32_t)(K0 >> 32); r0.x = (uint32_t)((K0 >> 3) & 0x1FFFFFull) + 1u; r0.y = (uint32_t)((K0 >> 24) & 0xFFull) * 8u + (uint32_t)(K0 & 7ull) + 1u;
        r1.score = (int32_t)(K1 >> 32); r1.x = (uint32_t)((K1 >> 3) & 0x1FFFFFull) + 1u; r1.y = (uint32_t)((K1 >> 24) & 0xFFull) * 8u + (uint32_t)(K1 & 7ull) + 1u;
    } else {
        uint32_t vM = V[1];
#pragma unroll
        for (int k = 2; k <= W; ++k) if ((uint32_t)k == km) vM = V[k];
        int32_t s0 = (TYPE == NVB_GLOBAL) ? half_lo(vM) - Go : ss0, s1 = (TYPE == NVB_GLOBAL) ? half_hi(vM) - Go : ss1;
        uint32_t x0 = (TYPE == NVB_GLOBAL) ? N : sx0, x1 = (TYPE == NVB_GLOBAL) ? N : sx1;
        s0 = __shfl_sync(FULL, s0, (int)(L - 1u)); s1 = __shfl_sync(FULL, s1, (int)(L - 1u));
        x0 = __shfl_sync(FULL, x0, (int)(L - 1u)); x1 = __shfl_sync(FULL, x1, (int)(L - 1u));
        r0.score = s0; r0.x = x0; r0.y = M; r1.score = s1; r1.x = x1; r1.y = M;
    }
    if (lane == 0u) {
        b.score[a0] = r0.score; b.sink[a0] = make_uint2(r0.x, r0.y);
        if (has1) { b.score[a1] = r1.score; b.sink[a1] = make_uint2(r1.x, r1.y); }
    }
}

// full-matrix traceback from KNOWN sinks, one warp per alignment (FullTbLane, gotoh_full_core.cuh): item i = (alignment a, output slot);
// a resident grid strides over the device-side item count, each warp owning one slot of `slot_words` direction words in `pool`.
// Only text rows [r0, sink.x) are computed (full_traceback_first_row); lane 0 then walks the step-major matrix from the sink, which
// the score pass already placed exactly where the reference does, so no LOCAL tie order is tracked here.
// (FullTbOut, full_warp_traceback: gotoh_full_core.cuh)

template <int TYPE, int W>
__global__ void __launch_bounds__(WARP_BLOCKDIM)
gotoh_full_warp_traceback_kernel(const GotohScheme S, const StrSet pat, const StrSet txt, const uint8_t* __restrict__ quals,
                                 const int32_t* __restrict__ score, const uint2* __restrict__ sink,
                                 const uint2* __restrict__ items, const uint32_t* __restrict__ n_items,
                                 const FullTbOut o, uint32_t* __restrict__ pool, const uint32_t slot_words)
{
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    constexpr int NW = FullTbLane<W>::NW;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = (blockIdx.x * WARP_BLOCKDIM + threadIdx.x) >> 5, n_warps = (gridDim.x * WARP_BLOCKDIM) >> 5;
    uint32_t* __restrict__ dirs = pool + (size_t)warp * slot_words;
    const int32_t INF = SHRT_MIN - (S.pgo < S.pge ? S.pgo : S.pge);
    // the largest substitution score (front cut of LOCAL windows)
    int32_t s_max = S.match > S.mismatch ? S.match : S.mismatch;
    if (S.qtab) {
        s_max = INT_MIN;
        for (uint32_t i = lane; i < 512u; i += 32u) s_max = imax2(s_max, S.qtab[i]);
        s_max = __reduce_max_sync(FULL, s_max);
    }
    const uint32_t n = *n_items;
    for (uint32_t i = warp; i < n; i += n_warps) {
        const uint2 it = items[i];
        const uint32_t a = it.x, out = it.y;
        const uint2 sk = sink[a];
        const uint32_t M = str_len(pat, a), c0 = lane * (uint32_t)W;
        const uint32_t r0 = full_traceback_first_row(TYPE, sk.x, sk.y, score[a], s_max, S.pgo, S.pge);
        const uint32_t R = sk.x - r0, L = (M + (uint32_t)W - 1u) / (uint32_t)W;
        const uint32_t toff = str_off(txt, a) + r0;
        FullTbLane<W> ln;
        ln.template init<TYPE>(S, pat.words, pat.bits, pat.big_endian, str_off(pat, a), M, quals, c0, INF);
        int32_t outH = 0, outE = 0;
        uint32_t outG = 0u, myG = 0u;
        const uint32_t steps = R + L - 1u;
        for (uint32_t t = 0; t < steps; ++t) {
            if ((t & 31u) == 0u) myG = (t + lane < R) ? sym_at_rt(txt.words, txt.bits, txt.big_endian, toff + t + lane) : 255u;
            const uint32_t rowG = __shfl_sync(FULL, myG, t & 31u);
            int32_t Hl = __shfl_up_sync(FULL, outH, 1), E = __shfl_up_sync(FULL, outE, 1);
            uint32_t g = __shfl_up_sync(FULL, outG, 1);
            const uint32_t r = t - lane;                                   // wraps for t < lane: then r >= R
            if (lane == 0u) { full_first_column<TYPE>(S, r0 + r, INF, Hl, E); g = rowG; }
            if (r < R && lane < L) {
                uint32_t dw[NW];
                ln.template row<TYPE>(S, g, Hl, E, dw);
                outH = Hl; outE = E; outG = g;
#pragma unroll
                for (int w = 0; w < NW; ++w) dirs[((size_t)t * NW + w) * 32u + lane] = dw[w];
            }
        }
        __syncwarp();
        if (lane == 0u) {
            SinkResult s; s.score = score[a]; s.x = R; s.y = sk.y;
            uint32_t sx = 0u, sy = 0u;
            const uint32_t cnt = gotoh_full_walk<TYPE>(FullDirsStepMajor{dirs, (uint32_t)W, (uint32_t)NW}, s, o.ops + (size_t)out * o.max_ops,
                                                       o.max_ops, sx, sy);
            o.source[out] = make_uint2((o.absolute ? str_off(txt, a) : 0u) + r0 + sx, sy);
            o.n_ops[out] = cnt;
        }
        __syncwarp();                                                      // the slot is rewritten by the next item
    }
}

// nvb_debug_full_traceback_warp: every alignment with a sink becomes an item (a, a); the others get no ops and source (-1, -1)
__global__ void __launch_bounds__(256)
full_tb_items_kernel(const uint32_t n, const uint2* __restrict__ sink, uint2* __restrict__ items, uint32_t* __restrict__ n_items,
                     uint32_t* __restrict__ n_ops, uint2* __restrict__ source)
{
    const uint32_t a = blockIdx.x * 256 + threadIdx.x;
    if (a >= n) return;
    const uint2 k = sink[a];
    if (k.x == 0xFFFFFFFFu || k.y == 0xFFFFFFFFu) { n_ops[a] = 0u; source[a] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu); return; }
    items[atomicAdd(n_items, 1u)] = make_uint2(a, a);
}

template <int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_full_todo_kernel(const GotohScheme S, const GotohBatch b, int2* __restrict__ col, const uint32_t* __restrict__ todo, const uint32_t* __restrict__ todo_count)
{
    const uint32_t n = *todo_count;
    for (uint32_t t = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x; t < n; t += gridDim.x * GENERIC_BLOCKDIM) {
        const uint32_t a = todo[t];
        const SinkResult r = gotoh_full<TYPE>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), str_len(b.pat, a),
                                              b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a),
                                              col + a, (size_t)b.n_max, b.quals);
        b.score[a] = r.score;
        b.sink[a]  = make_uint2(r.x, r.y);
    }
}

// traceback: one alignment per thread; DP with direction vectors into a per-alignment global scratch matrix
// (M rows x DirWords<B>::N words -- no checkpoints / recomputation: 2.4 KB per 150 x 31 alignment is nothing in 80 GB),
// then the H/E/F state-machine walk from the sink.

// todo != NULL: only the alignments listed there (those the gapless fast path could not resolve), todo_count on the device
template <int B, int TYPE>
__global__ void __launch_bounds__(GENERIC_BLOCKDIM)
gotoh_traceback_kernel(const GotohScheme S, const GotohBatch b, const TracebackOut o, const uint32_t* __restrict__ todo, const uint32_t* __restrict__ todo_count)
{
    constexpr int NW = DirWords<B>::N;
    const uint32_t n = todo ? *todo_count : batch_count(b);
    for (uint32_t i = blockIdx.x * GENERIC_BLOCKDIM + threadIdx.x; i < n; i += gridDim.x * GENERIC_BLOCKDIM) {
    const uint32_t a = todo ? todo[i] : i;
    uint32_t* dirs = o.dirs + (size_t)a * o.dir_rows * NW;
    const uint32_t M = str_len(b.pat, a);
    SinkResult r; r.score = NVB_SINK_MIN; r.x = r.y = 0xFFFFFFFFu;
    if (M <= o.dir_rows)
        r = gotoh_generic_impl<B, TYPE, true>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), M, b.quals,
                                              b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a), dirs);
    b.score[a] = r.score;
    b.sink[a]  = make_uint2(r.x, r.y);
    uint32_t sx = 0xFFFFFFFFu, sy = 0xFFFFFFFFu, cnt = 0;
    if (r.x != 0xFFFFFFFFu && r.y != 0xFFFFFFFFu)
        cnt = gotoh_walk<B, TYPE>(dirs, r, o.ops + (size_t)a * o.max_ops, o.max_ops, sx, sy);
    o.source[a] = make_uint2(sx, sy);
    o.n_ops[a]  = cnt;
    }
}

// gapless fast path (gapless_traceback, gotoh_core.cuh): score and sink are already in b.score / b.sink (from the score kernels); the
// alignments it resolves get their source, op count and all-substitution op string, the others are appended to the todo list
template <int TYPE>
__global__ void __launch_bounds__(256)
gotoh_traceback_gapless_kernel(const GotohScheme S, const GotohBatch b, const TracebackOut o, uint32_t* __restrict__ todo, uint32_t* __restrict__ todo_count)
{
    const uint32_t a = blockIdx.x * 256 + threadIdx.x;
    const bool in_range = a < batch_count(b);
    uint32_t len = 0u;
    bool done = false;
    if (in_range) {
        const uint2 k = b.sink[a];
        done = gapless_traceback<TYPE>(S, b.pat.words, b.pat.bits, b.pat.big_endian, str_off(b.pat, a), str_len(b.pat, a), b.quals,
                                       b.txt.words, b.txt.bits, b.txt.big_endian, str_off(b.txt, a), str_len(b.txt, a), b.score[a], k.x, k.y, len);
        if (done) {
            o.source[a] = make_uint2(k.x - len, k.y - len);
            o.n_ops[a]  = len;
        } else {
            todo[atomicAdd(todo_count, 1u)] = a;
        }
    }
    // the op strings, a warp per row: 32 consecutive bytes per store instead of 32 rows touched by each
    const uint32_t lane = threadIdx.x & 31u, a0 = a - lane;
    const uint32_t wrote = __ballot_sync(0xffffffffu, done);
    for (uint32_t w = wrote; w; w &= w - 1u) {
        const uint32_t src = __ffs(w) - 1u;
        uint32_t m = __shfl_sync(0xffffffffu, len, src);
        m = m < o.max_ops ? m : o.max_ops;
        uint8_t* ops = o.ops + (size_t)(a0 + src) * o.max_ops;
        for (uint32_t i = lane; i < m; i += 32u) ops[i] = (uint8_t)DIR_SUB;
    }
}

template <int B, int TYPE>
static int launch_traceback(const GotohScheme& S, const GotohBatch& b, const TracebackOut& o, const uint32_t* todo, const uint32_t* todo_count, cudaStream_t s)
{
    // (with a todo list the count lives on the device: the grid is sized for the whole batch and the surplus CTAs leave at once --
    // a capped, striding grid left most of the SMs' thread slots empty when only a minority of the alignments is listed)
    const uint32_t grid = (b.n_max + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM;
    gotoh_traceback_kernel<B, TYPE><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, o, todo, todo_count);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

template <int B, int TYPE>
static int launch_generic(const GotohScheme& S, const GotohBatch& b, const uint32_t* todo, const uint32_t* todo_count, uint32_t n_hint, cudaStream_t s)
{
    // grid-stride: the count may live on the device
    uint32_t grid = (n_hint + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM;
    const uint32_t cap = sm_count() * 32u;
    if (todo) grid = grid < cap ? grid : cap;
    if (grid == 0) grid = 1;
    gotoh_generic_kernel<B, TYPE><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, todo, todo_count);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

template <int B, int TYPE, int PFMT, bool ROWS2, bool TICKET>
static int launch_pair_grid(const GotohScheme& S, const GotohBatch& b, uint32_t sel_rows, uint32_t* todo, uint32_t* todo_count, cudaStream_t s)
{
    const size_t smem = (size_t)((sel_rows + 15u) & ~15u) * PAIR_BLOCKDIM * sizeof(uint16_t) + (size_t)g_pair_extra_smem;   // whole words of 16 columns
    // the attribute is per DEVICE: a host that drives several GPUs from one process (nvBowtie's one compute thread per
    // device) must set it on each; one atomic flag per (instantiation, device)
    static std::atomic<bool> attr_done[NVB_MAX_DEVICES];
    int dev = 0;
    NVB_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= NVB_MAX_DEVICES) return NVB_E_UNSUPPORTED;
    if (!attr_done[dev].load(std::memory_order_acquire)) {
        NVB_CUDA_TRY(cudaFuncSetAttribute(gotoh_pair_kernel<B, TYPE, PFMT, ROWS2, TICKET>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done[dev].store(true, std::memory_order_release);
    }
    const uint32_t pairs = (b.n_max + 1u) / 2u;
    uint32_t grid = (pairs + PAIR_BLOCKDIM - 1) / PAIR_BLOCKDIM;
    if (TICKET) {                                                  // resident: what the SMs hold at once
        int per_sm = 0;
        NVB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gotoh_pair_kernel<B, TYPE, PFMT, ROWS2, TICKET>, PAIR_BLOCKDIM, smem));
        const uint32_t resident = sm_count() * (uint32_t)(per_sm > 0 ? per_sm : 1);
        grid = grid < resident ? grid : resident;
    }
    gotoh_pair_kernel<B, TYPE, PFMT, ROWS2, TICKET><<<grid, PAIR_BLOCKDIM, smem, s>>>(S, b, sel_rows, todo, todo_count);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}
template <int B, int TYPE, int PFMT, bool ROWS2>
static int launch_pair_fmt(const GotohScheme& S, const GotohBatch& b, uint32_t sel_rows, uint32_t* todo, uint32_t* todo_count, cudaStream_t s)
{
    if (b.d_n) return launch_pair_grid<B, TYPE, PFMT, ROWS2, true>(S, b, sel_rows, todo, todo_count, s);
    return launch_pair_grid<B, TYPE, PFMT, ROWS2, false>(S, b, sel_rows, todo, todo_count, s);
}
template <int B, int TYPE, int PFMT>
static int launch_pair_rows(const GotohScheme& S, const GotohBatch& b, uint32_t sel_rows, uint32_t* todo, uint32_t* todo_count, cudaStream_t s)
{
    if (g_pair_rows2) return launch_pair_fmt<B, TYPE, PFMT, true>(S, b, sel_rows, todo, todo_count, s);
    return launch_pair_fmt<B, TYPE, PFMT, false>(S, b, sel_rows, todo, todo_count, s);
}
// pattern format known at compile time (2- / 4-bit big-endian, no quality table): the specialised kernels; anything else: PFMT 0
template <int B, int TYPE>
static int launch_pair(const GotohScheme& S, const GotohBatch& b, uint32_t sel_rows, uint32_t* todo, uint32_t* todo_count, cudaStream_t s)
{
    if (!S.qtab && b.pat.big_endian && b.pat.bits == 2u && g_pair_fmt_ok) return launch_pair_rows<B, TYPE, 2>(S, b, sel_rows, todo, todo_count, s);
    if (!S.qtab && b.pat.big_endian && b.pat.bits == 4u && g_pair_fmt_ok) return launch_pair_rows<B, TYPE, 4>(S, b, sel_rows, todo, todo_count, s);
    return launch_pair_rows<B, TYPE, 0>(S, b, sel_rows, todo, todo_count, s);
}

#define NVB_TYPE_SWITCH(BAND, FN, ...)                                            \
    switch (type) {                                                               \
    case NVB_GLOBAL:      return FN<BAND, NVB_GLOBAL>(__VA_ARGS__);               \
    case NVB_LOCAL:       return FN<BAND, NVB_LOCAL>(__VA_ARGS__);                \
    case NVB_SEMI_GLOBAL: return FN<BAND, NVB_SEMI_GLOBAL>(__VA_ARGS__);          \
    default:              return NVB_E_INVALID; }

static int dispatch_generic(int band, int type, const GotohScheme& S, const GotohBatch& b, const uint32_t* todo, const uint32_t* todo_count, uint32_t n_hint, cudaStream_t s)
{
    switch (band) {
    case 3:  NVB_TYPE_SWITCH(3,  launch_generic, S, b, todo, todo_count, n_hint, s)
    case 5:  NVB_TYPE_SWITCH(5,  launch_generic, S, b, todo, todo_count, n_hint, s)
    case 7:  NVB_TYPE_SWITCH(7,  launch_generic, S, b, todo, todo_count, n_hint, s)
    case 15: NVB_TYPE_SWITCH(15, launch_generic, S, b, todo, todo_count, n_hint, s)
    case 31: NVB_TYPE_SWITCH(31, launch_generic, S, b, todo, todo_count, n_hint, s)
    case 63: NVB_TYPE_SWITCH(63, launch_generic, S, b, todo, todo_count, n_hint, s)
    }
    return NVB_E_INVALID;
}
static int dispatch_pair(int band, int type, const GotohScheme& S, const GotohBatch& b, uint32_t sel_rows, uint32_t* todo, uint32_t* todo_count, cudaStream_t s)
{
    switch (band) {
    case 7:  NVB_TYPE_SWITCH(7,  launch_pair, S, b, sel_rows, todo, todo_count, s)
    case 15: NVB_TYPE_SWITCH(15, launch_pair, S, b, sel_rows, todo, todo_count, s)
    case 31: NVB_TYPE_SWITCH(31, launch_pair, S, b, sel_rows, todo, todo_count, s)
    }
    return NVB_E_INVALID;
}

static int dispatch_traceback(int band, int type, const GotohScheme& S, const GotohBatch& b, const TracebackOut& o, const uint32_t* todo, const uint32_t* todo_count, cudaStream_t s)
{
    switch (band) {
    case 3:  NVB_TYPE_SWITCH(3,  launch_traceback, S, b, o, todo, todo_count, s)
    case 5:  NVB_TYPE_SWITCH(5,  launch_traceback, S, b, o, todo, todo_count, s)
    case 7:  NVB_TYPE_SWITCH(7,  launch_traceback, S, b, o, todo, todo_count, s)
    case 15: NVB_TYPE_SWITCH(15, launch_traceback, S, b, o, todo, todo_count, s)
    case 31: NVB_TYPE_SWITCH(31, launch_traceback, S, b, o, todo, todo_count, s)
    }
    return NVB_E_INVALID;
}
static inline int dir_words(int band) { return (band * 4 + 31) / 32; }

// force_path: 0 auto, 1 generic only (used by tests to exercise both paths on the same inputs)
static int g_force_path = 0;
static int g_full_warp = 0;           // 0 = by batch size, 1 = always the warp-per-pair kernel, 2 = never (nvb_debug_full_warp)
static uint32_t g_full_warp_max_pairs = 30000u;   // measured cross-over with the thread-per-pair kernel: ~50-60 K alignments
static int g_full_minb = 0;          // 0 = per-type default; tuning knob of gotoh_full_pair_kernel's occupancy (nvb_debug_full_minb)
// route of the last banded / full-matrix score call (nvb_debug_gotoh_last_route): 0 = no packed kernel, 1 = pair kernel, 2 = warp
// kernel, and the todo-list count of that call (in the caller's temp buffer)
static int g_route_packed = 0;
static const uint32_t* g_route_todo_count = nullptr;
static void set_route(int packed, const uint32_t* todo_count) { g_route_packed = packed; g_route_todo_count = todo_count; }

static int banded_impl(int band, int type, const nvb_gotoh_scheme* scheme,
                       const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts,
                       const uint32_t* d_n, uint32_t n_max, int32_t* d_score, nvb_uint2* d_sink,
                       void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!scheme || !temp_bytes || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (!(band == 3 || band == 5 || band == 7 || band == 15 || band == 31 || band == 63)) return NVB_E_INVALID;
    if (type < 0 || type > 2) return NVB_E_INVALID;

    TempCarver tc(d_temp);
    uint32_t* todo_count = tc.take<uint32_t>(4);
    uint32_t* todo       = tc.take<uint32_t>((size_t)n_max + 2);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n_max == 0) return NVB_OK;
    if (!d_score || !d_sink) return NVB_E_INVALID;

    cudaStream_t s = as_stream(stream);
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = d_n; b.n_max = n_max; b.score = d_score; b.sink = (uint2*)d_sink;
    const GotohScheme S = make_scheme(scheme);

    // `length` is the maximum pattern length (the reference's batch API takes max_pattern_length too,
    // nvbio/alignment/batched_inl.h:1067-1101)
    const uint32_t max_m = patterns->length;
    const uint32_t sel_rows = max_m + (uint32_t)band - 1u;
    const size_t smem = (size_t)((sel_rows + 15u) & ~15u) * PAIR_BLOCKDIM * sizeof(uint16_t);          // as launch_pair_fmt sizes it (two-byte selectors)
    const bool fast = (g_force_path != 1) && texts->bits == 2 && max_m >= 1 && smem <= 200u * 1024u &&
                      pair_path_ok(band, type, scheme, max_m);
    if (!fast) { set_route(0, nullptr); return dispatch_generic(band, type, S, b, nullptr, nullptr, n_max, s); }

    set_route(1, todo_count);
    NVB_CUDA_TRY(cudaMemsetAsync(todo_count, 0, 2 * sizeof(uint32_t), s));     // [0] the todo list's length, [1] the pair ticket
    int r = dispatch_pair(band, type, S, b, sel_rows, todo, todo_count, s);
    if (r != NVB_OK) return r;
    return dispatch_generic(band, type, S, b, todo, todo_count, n_max, s);
}

// the warp traceback's launch: a resident grid (its measured occupancy times the SM count), one pool slot per warp
template <int TYPE, int W>
static int full_tb_launch(const FullTbArgs* a, uint32_t max_n, size_t* pool_bytes, cudaStream_t s)
{
    int per_sm = 0;
    NVB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gotoh_full_warp_traceback_kernel<TYPE, W>, WARP_BLOCKDIM, 0));
    const uint32_t grid = sm_count() * (uint32_t)(per_sm > 0 ? per_sm : 1);
    const uint32_t slot_words = (max_n + 31u) * 32u * (uint32_t)FullTbLane<W>::NW;
    *pool_bytes = (size_t)grid * (WARP_BLOCKDIM / 32) * slot_words * sizeof(uint32_t);
    if (!a) return NVB_OK;
    gotoh_full_warp_traceback_kernel<TYPE, W><<<grid, WARP_BLOCKDIM, 0, s>>>(a->S, a->pat, a->txt, a->quals, a->score, a->sink, a->items,
                                                                            a->n_items, a->o, (uint32_t*)a->pool, slot_words);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int full_warp_traceback(int type, uint32_t max_m, uint32_t max_n, const FullTbArgs* a, size_t* pool_bytes, cudaStream_t s)
{
    if (max_m < 1u || max_m > FULL_TB_MAX_M || max_n > 65535u) return NVB_E_UNSUPPORTED;
#define NVB_TB_W(T)                                                                                                                 \
    switch ((max_m + 31u) / 32u) {                                                                                                  \
    case 1:  return full_tb_launch<T, 1>(a, max_n, pool_bytes, s);  case 2:  return full_tb_launch<T, 2>(a, max_n, pool_bytes, s);   \
    case 3:  return full_tb_launch<T, 3>(a, max_n, pool_bytes, s);  case 4:  return full_tb_launch<T, 4>(a, max_n, pool_bytes, s);   \
    case 5:  return full_tb_launch<T, 5>(a, max_n, pool_bytes, s);  case 6:  return full_tb_launch<T, 6>(a, max_n, pool_bytes, s);   \
    case 7:  return full_tb_launch<T, 7>(a, max_n, pool_bytes, s);  case 8:  return full_tb_launch<T, 8>(a, max_n, pool_bytes, s);   \
    case 9:  return full_tb_launch<T, 9>(a, max_n, pool_bytes, s);  case 10: return full_tb_launch<T, 10>(a, max_n, pool_bytes, s);  \
    case 11: return full_tb_launch<T, 11>(a, max_n, pool_bytes, s); case 12: return full_tb_launch<T, 12>(a, max_n, pool_bytes, s);  \
    case 13: return full_tb_launch<T, 13>(a, max_n, pool_bytes, s); case 14: return full_tb_launch<T, 14>(a, max_n, pool_bytes, s);  \
    case 15: return full_tb_launch<T, 15>(a, max_n, pool_bytes, s); default: return full_tb_launch<T, 16>(a, max_n, pool_bytes, s); }
    switch (type) {
    case NVB_GLOBAL: NVB_TB_W(NVB_GLOBAL)
    case NVB_LOCAL:  NVB_TB_W(NVB_LOCAL)
    default:         NVB_TB_W(NVB_SEMI_GLOBAL)
    }
#undef NVB_TB_W
}

} // namespace nvb

using namespace nvb;

extern "C" {

int nvb_banded_gotoh_score(int band_len, int type, const nvb_gotoh_scheme* scheme,
                           const nvb_string_set* patterns, const uint8_t* d_quals,
                           const nvb_string_set* texts, uint32_t n,
                           int32_t* d_score, nvb_uint2* d_sink,
                           void* d_temp, size_t* temp_bytes, void* stream)
{
    return banded_impl(band_len, type, scheme, patterns, d_quals, texts, nullptr, n, d_score, d_sink, d_temp, temp_bytes, stream);
}

int nvb_banded_gotoh_score_indirect(int band_len, int type, const nvb_gotoh_scheme* scheme,
                           const nvb_string_set* patterns, const uint8_t* d_quals,
                           const nvb_string_set* texts, const uint32_t* d_n, uint32_t n_max,
                           int32_t* d_score, nvb_uint2* d_sink,
                           void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!d_n) return NVB_E_INVALID;
    return banded_impl(band_len, type, scheme, patterns, d_quals, texts, d_n, n_max, d_score, d_sink, d_temp, temp_bytes, stream);
}

static int gotoh_full_impl(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts,
                           const uint32_t* d_n, uint32_t n,
                           int32_t* d_score, nvb_uint2* d_sink, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!scheme || !temp_bytes || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (type < 0 || type > 2) return NVB_E_INVALID;
    if (texts->length > 65535u || patterns->length > 65535u) return NVB_E_UNSUPPORTED;
    TempCarver tc(d_temp);
    const bool need_col = patterns->length > (uint32_t)FULL_W;          // a single stripe needs no boundary column
    int2* col = need_col ? tc.take<int2>((size_t)(n + 1u) * (texts->length ? texts->length : 1u)) : tc.take<int2>(1);
    uint32_t* todo_count = tc.take<uint32_t>(4);
    uint32_t* todo       = tc.take<uint32_t>((size_t)n + 2);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n == 0) return NVB_OK;
    if (!d_score || !d_sink) return NVB_E_INVALID;
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = d_n; b.n_max = n; b.score = d_score; b.sink = (uint2*)d_sink;
    const GotohScheme S = make_scheme(scheme);
    const uint32_t grid = (n + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM;
    cudaStream_t s = as_stream(stream);
    const bool packed = g_force_path != 1 && full_pair_path_ok(type, scheme, patterns->length, texts->length);
    if (!packed) {
        set_route(0, nullptr);
        switch (type) {
        case NVB_GLOBAL:      gotoh_full_kernel<NVB_GLOBAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col); break;
        case NVB_LOCAL:       gotoh_full_kernel<NVB_LOCAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col); break;
        default:              gotoh_full_kernel<NVB_SEMI_GLOBAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col); break;
        }
        NVB_LAUNCH_CHECK();
        return NVB_OK;
    }
    // packed pairs first (the boundary columns of pair p live in the first half of `col`), then whatever they rejected
    NVB_CUDA_TRY(cudaMemsetAsync(todo_count, 0, sizeof(uint32_t), s));
    const uint32_t n_pairs = (n + 1u) >> 1;
    // small batches: one warp per pair (a thread per pair would leave most of the SMs idle); W columns per lane
    const uint32_t max_m = patterns->length;
    // with a device-side count (`n` is then only a capacity) the batch is usually much smaller than its capacity: allow 4x
    const bool use_warp = g_full_warp == 1 || (g_full_warp == 0 && n_pairs <= (d_n ? 4u : 1u) * g_full_warp_max_pairs);
    if (use_warp && max_m >= 1u && max_m <= 256u && !S.qtab) {           // (the warp kernel has no quality-table form)
        set_route(2, todo_count);
        const uint32_t Wc = (max_m + 31u) / 32u;
        const uint32_t wgrid = (uint32_t)(((uint64_t)n_pairs * 32u + WARP_BLOCKDIM - 1) / WARP_BLOCKDIM);
        const uint32_t tgrid2 = grid < sm_count() * 8u ? grid : sm_count() * 8u;
#define NVB_FULL_WARP_W(T, WW) gotoh_full_warp_kernel<T, WW><<<wgrid, WARP_BLOCKDIM, 0, s>>>(S, b, todo, todo_count)
#define NVB_FULL_WARP(T)                                                                                   \
        switch (Wc) {                                                                                      \
        case 1: NVB_FULL_WARP_W(T, 1); break; case 2: NVB_FULL_WARP_W(T, 2); break;                        \
        case 3: NVB_FULL_WARP_W(T, 3); break; case 4: NVB_FULL_WARP_W(T, 4); break;                        \
        case 5: NVB_FULL_WARP_W(T, 5); break; case 6: NVB_FULL_WARP_W(T, 6); break;                        \
        case 7: NVB_FULL_WARP_W(T, 7); break; default: NVB_FULL_WARP_W(T, 8); break; }                     \
        gotoh_full_todo_kernel<T><<<tgrid2, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, todo, todo_count);
        switch (type) {
        case NVB_GLOBAL: NVB_FULL_WARP(NVB_GLOBAL) break;
        case NVB_LOCAL:  NVB_FULL_WARP(NVB_LOCAL) break;
        default:         NVB_FULL_WARP(NVB_SEMI_GLOBAL) break;
        }
#undef NVB_FULL_WARP
#undef NVB_FULL_WARP_W
        NVB_LAUNCH_CHECK();
        return NVB_OK;
    }
    set_route(1, todo_count);
    const uint32_t pgrid = (n_pairs + PAIR_BLOCKDIM - 1) / PAIR_BLOCKDIM;
    uint32_t tgrid = grid < sm_count() * 8u ? grid : sm_count() * 8u;
    // occupancy: with two text rows in flight every type fits spill-free at 2 CTAs per SM (210-250 registers); tools/bench_full.py
    // sweeps the alternatives (nvb_debug_full_minb)
    const int minb = g_full_minb ? g_full_minb : 2;
#define NVB_FULL_PAIR(T)                                                                                               \
    if (minb == 2)      gotoh_full_pair_kernel<T, 2><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); \
    else if (minb == 4)        gotoh_full_pair_kernel<T, 4><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); \
    else                       gotoh_full_pair_kernel<T, 3><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); \
    gotoh_full_todo_kernel<T><<<tgrid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, todo, todo_count);
    if (S.qtab) {
        // quality-dependent scores: per-column profiles (32 KB of shared memory per CTA), 2 CTAs per SM
        switch (type) {
        case NVB_GLOBAL: gotoh_full_pair_kernel<NVB_GLOBAL, 2, true><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); break;
        case NVB_LOCAL:  gotoh_full_pair_kernel<NVB_LOCAL, 2, true><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); break;
        default:         gotoh_full_pair_kernel<NVB_SEMI_GLOBAL, 2, true><<<pgrid, PAIR_BLOCKDIM, 0, s>>>(S, b, (uint2*)col, todo, todo_count); break;
        }
        switch (type) {
        case NVB_GLOBAL: gotoh_full_todo_kernel<NVB_GLOBAL><<<tgrid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, todo, todo_count); break;
        case NVB_LOCAL:  gotoh_full_todo_kernel<NVB_LOCAL><<<tgrid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, todo, todo_count); break;
        default:         gotoh_full_todo_kernel<NVB_SEMI_GLOBAL><<<tgrid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, todo, todo_count); break;
        }
        NVB_LAUNCH_CHECK();
        return NVB_OK;
    }
    switch (type) {
    case NVB_GLOBAL: NVB_FULL_PAIR(NVB_GLOBAL) break;
    case NVB_LOCAL:  NVB_FULL_PAIR(NVB_LOCAL) break;
    default:         NVB_FULL_PAIR(NVB_SEMI_GLOBAL) break;
    }
#undef NVB_FULL_PAIR
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_gotoh_score(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                    int32_t* d_score, nvb_uint2* d_sink, void* d_temp, size_t* temp_bytes, void* stream)
{
    return gotoh_full_impl(type, scheme, patterns, d_quals, texts, nullptr, n, d_score, d_sink, d_temp, temp_bytes, stream);
}

int nvb_gotoh_score_indirect(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts,
                             const uint32_t* d_n, uint32_t n_max,
                             int32_t* d_score, nvb_uint2* d_sink, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!d_n) return NVB_E_INVALID;
    return gotoh_full_impl(type, scheme, patterns, d_quals, texts, d_n, n_max, d_score, d_sink, d_temp, temp_bytes, stream);
}

} // extern "C"

namespace nvb {
int banded_traceback(int band_len, int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals,
                     const nvb_string_set* texts, const uint32_t* d_n, uint32_t n, int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                     uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!scheme || !temp_bytes || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (!(band_len == 3 || band_len == 5 || band_len == 7 || band_len == 15 || band_len == 31)) return NVB_E_INVALID;
    if (type < 0 || type > 2) return NVB_E_INVALID;
    const uint32_t max_m = patterns->length ? patterns->length : 1u;
    TempCarver tc(d_temp);
    uint32_t* dirs = tc.take<uint32_t>((size_t)n * max_m * dir_words(band_len));
    uint32_t* todo_count = tc.take<uint32_t>(4);
    uint32_t* todo       = tc.take<uint32_t>((size_t)n + 2);
    size_t score_bytes = 0;                                   // scratch of the score pass, carved behind the rest
    {
        const int r = banded_impl(band_len, type, scheme, patterns, d_quals, texts, nullptr, n, nullptr, nullptr, nullptr, &score_bytes, nullptr);
        if (r != NVB_E_TEMP_SIZE && r != NVB_OK) return r;
    }
    char* score_tmp = tc.take<char>(score_bytes + 256);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n == 0) return NVB_OK;
    if (!d_score || !d_sink || !d_source || !d_ops || !d_n_ops || max_ops == 0) return NVB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = d_n; b.n_max = n; b.score = d_score; b.sink = (uint2*)d_sink;
    TracebackOut o;
    o.source = (uint2*)d_source; o.ops = d_ops; o.n_ops = d_n_ops; o.max_ops = max_ops; o.dirs = dirs; o.dir_rows = max_m;
    const GotohScheme S = make_scheme(scheme);
    if (!g_traceback_fast || type == NVB_GLOBAL) {
        set_route(0, nullptr);
        return dispatch_traceback(band_len, type, S, b, o, nullptr, nullptr, s);
    }
    // 1. score + sink with the score kernels (DPX where admitted); 2. the gapless fast path resolves every alignment whose optimal path
    // has no gap (most reads) from the sink alone; 3. the rest goes through the direction-matrix traceback
    {
        size_t sb = score_bytes + 256;
        const int r = banded_impl(band_len, type, scheme, patterns, d_quals, texts, d_n, n, d_score, d_sink, score_tmp, &sb, stream);
        if (r != NVB_OK) return r;
    }
    NVB_CUDA_TRY(cudaMemsetAsync(todo_count, 0, sizeof(uint32_t), s));
    if (type == NVB_LOCAL) gotoh_traceback_gapless_kernel<NVB_LOCAL><<<(n + 255u) / 256u, 256, 0, s>>>(S, b, o, todo, todo_count);
    else                   gotoh_traceback_gapless_kernel<NVB_SEMI_GLOBAL><<<(n + 255u) / 256u, 256, 0, s>>>(S, b, o, todo, todo_count);
    NVB_LAUNCH_CHECK();
    return dispatch_traceback(band_len, type, S, b, o, todo, todo_count, s);
}
} // namespace nvb

extern "C" {

int nvb_banded_gotoh_traceback(int band_len, int type, const nvb_gotoh_scheme* scheme,
                               const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                               int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                               uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops,
                               void* d_temp, size_t* temp_bytes, void* stream)
{
    return banded_traceback(band_len, type, scheme, patterns, d_quals, texts, nullptr, n, d_score, d_sink, d_source, d_ops, max_ops, d_n_ops,
                            d_temp, temp_bytes, stream);
}

int nvb_banded_gotoh_score_window(int band_len, int type, const nvb_gotoh_scheme* scheme,
                                  const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                                  uint32_t window_begin, uint32_t window_end, const int32_t* d_min_score,
                                  int16_t* d_checkpoints, int32_t* d_score, nvb_uint2* d_sink, uint8_t* d_alive, void* stream)
{
    if (!scheme || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (type < 0 || type > 2 || window_begin >= window_end) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    if (!d_checkpoints || !d_score || !d_sink || !d_alive) return NVB_E_INVALID;
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = nullptr; b.n_max = n; b.score = d_score; b.sink = (uint2*)d_sink;
    WindowArgs w; w.wb = window_begin; w.we = window_end; w.min_score = d_min_score; w.ckpt = (short2*)d_checkpoints; w.alive = d_alive;
    const GotohScheme S = make_scheme(scheme);
    cudaStream_t s = as_stream(stream);
    switch (band_len) {
    case 3:  NVB_TYPE_SWITCH(3,  launch_window, S, b, w, s)
    case 5:  NVB_TYPE_SWITCH(5,  launch_window, S, b, w, s)
    case 7:  NVB_TYPE_SWITCH(7,  launch_window, S, b, w, s)
    case 15: NVB_TYPE_SWITCH(15, launch_window, S, b, w, s)
    case 31: NVB_TYPE_SWITCH(31, launch_window, S, b, w, s)
    default: return NVB_E_INVALID;
    }
}

int nvb_banded_gotoh_score_best2(int band_len, int type, const nvb_gotoh_scheme* scheme,
                                 const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                                 uint32_t distinct_dist, int32_t* d_out6, void* stream)
{
    if (!scheme || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (type < 0 || type > 2) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    if (!d_out6) return NVB_E_INVALID;
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = nullptr; b.n_max = n; b.score = nullptr; b.sink = nullptr;
    const GotohScheme S = make_scheme(scheme);
    cudaStream_t s = as_stream(stream);
    switch (band_len) {
    case 3:  NVB_TYPE_SWITCH(3,  launch_best2, S, b, distinct_dist, d_out6, s)
    case 5:  NVB_TYPE_SWITCH(5,  launch_best2, S, b, distinct_dist, d_out6, s)
    case 7:  NVB_TYPE_SWITCH(7,  launch_best2, S, b, distinct_dist, d_out6, s)
    case 15: NVB_TYPE_SWITCH(15, launch_best2, S, b, distinct_dist, d_out6, s)
    case 31: NVB_TYPE_SWITCH(31, launch_best2, S, b, distinct_dist, d_out6, s)
    case 63: NVB_TYPE_SWITCH(63, launch_best2, S, b, distinct_dist, d_out6, s)
    default: return NVB_E_INVALID;
    }
}

static int g_full_tb_warp = 0;        // nvb_debug_full_traceback_warp(1): nvb_gotoh_traceback as the score dispatch + the warp traceback

// nvb_gotoh_traceback with nvb_debug_full_traceback_warp(1): score + sink from the score dispatch, then gotoh_full_warp_traceback_kernel
// from those sinks (its slot pool and window cuts) -- the path the paired-end traceback takes for rescued mates
static int gotoh_traceback_warp(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals,
                                const nvb_string_set* texts, uint32_t n, int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                                uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops, void* d_temp, size_t* temp_bytes, void* stream)
{
    cudaStream_t s = as_stream(stream);
    size_t score_bytes = 0, pool_bytes = 0;
    {
        const int r = gotoh_full_impl(type, scheme, patterns, d_quals, texts, nullptr, n, nullptr, nullptr, nullptr, &score_bytes, nullptr);
        if (r != NVB_E_TEMP_SIZE && r != NVB_OK) return r;
    }
    { const int r = full_warp_traceback(type, patterns->length, texts->length, nullptr, &pool_bytes, s); if (r != NVB_OK) return r; }
    TempCarver tc(d_temp);
    char* score_tmp = tc.take<char>(score_bytes);
    uint2* items = tc.take<uint2>(n ? n : 1u);
    uint32_t* n_items = tc.take<uint32_t>(4);
    void* pool = tc.take<char>(pool_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n == 0) return NVB_OK;
    if (!d_score || !d_sink || !d_source || !d_ops || !d_n_ops || max_ops == 0) return NVB_E_INVALID;
    {
        size_t sb = score_bytes;
        const int r = gotoh_full_impl(type, scheme, patterns, d_quals, texts, nullptr, n, d_score, d_sink, score_tmp, &sb, stream);
        if (r != NVB_OK) return r;
    }
    NVB_CUDA_TRY(cudaMemsetAsync(n_items, 0, sizeof(uint32_t), s));
    full_tb_items_kernel<<<(n + 255u) / 256u, 256, 0, s>>>(n, (const uint2*)d_sink, items, n_items, d_n_ops, (uint2*)d_source);
    NVB_LAUNCH_CHECK();
    FullTbArgs a;
    a.S = make_scheme(scheme); a.pat = make_strset(patterns); a.txt = make_strset(texts); a.quals = d_quals;
    a.score = d_score; a.sink = (const uint2*)d_sink; a.items = items; a.n_items = n_items;
    a.o.ops = d_ops; a.o.n_ops = d_n_ops; a.o.source = (uint2*)d_source; a.o.max_ops = max_ops; a.o.absolute = 0u;
    a.pool = pool;
    return full_warp_traceback(type, patterns->length, texts->length, &a, &pool_bytes, s);
}

int nvb_gotoh_traceback(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                        int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                        uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops,
                        void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!scheme || !temp_bytes || !valid_strset(patterns) || !valid_strset(texts)) return NVB_E_INVALID;
    if (type < 0 || type > 2) return NVB_E_INVALID;
    if (texts->length > 65535u || patterns->length > 65535u) return NVB_E_UNSUPPORTED;
    if (g_full_tb_warp == 1)
        return gotoh_traceback_warp(type, scheme, patterns, d_quals, texts, n, d_score, d_sink, d_source, d_ops, max_ops, d_n_ops, d_temp, temp_bytes, stream);
    const uint32_t max_m = patterns->length ? patterns->length : 1u, max_n = texts->length ? texts->length : 1u;
    const uint32_t dir_row_words = (max_m + 31u) / 32u * 4u;
    TempCarver tc(d_temp);
    int2* col = tc.take<int2>((size_t)n * max_n);
    uint32_t* dirs = tc.take<uint32_t>((size_t)n * max_n * dir_row_words);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n == 0) return NVB_OK;
    if (!d_score || !d_sink || !d_source || !d_ops || !d_n_ops || max_ops == 0) return NVB_E_INVALID;
    GotohBatch b;
    b.pat = make_strset(patterns); b.txt = make_strset(texts); b.quals = d_quals;
    b.d_n = nullptr; b.n_max = n; b.score = d_score; b.sink = (uint2*)d_sink;
    TracebackOut o;
    o.source = (uint2*)d_source; o.ops = d_ops; o.n_ops = d_n_ops; o.max_ops = max_ops; o.dirs = dirs; o.dir_rows = max_n;
    const GotohScheme S = make_scheme(scheme);
    const uint32_t grid = (n + GENERIC_BLOCKDIM - 1) / GENERIC_BLOCKDIM;
    cudaStream_t s = as_stream(stream);
    set_route(0, nullptr);
    switch (type) {
    case NVB_GLOBAL: gotoh_full_traceback_kernel<NVB_GLOBAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, o, dir_row_words); break;
    case NVB_LOCAL:  gotoh_full_traceback_kernel<NVB_LOCAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, o, dir_row_words); break;
    default:         gotoh_full_traceback_kernel<NVB_SEMI_GLOBAL><<<grid, GENERIC_BLOCKDIM, 0, s>>>(S, b, col, o, dir_row_words); break;
    }
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

// test / tuning hooks (include/nvbio_b200_debug.h)
void nvb_debug_force_gotoh_path(int path) { g_force_path = path; }
void nvb_debug_full_minb(int minb) { g_full_minb = minb; }
void nvb_debug_full_warp(int mode) { g_full_warp = mode; }
void nvb_debug_full_traceback_warp(int on) { g_full_tb_warp = on; }
void nvb_debug_pair_rows2(int on) { nvb::g_pair_rows2 = on; }
void nvb_debug_traceback_fast(int on) { nvb::g_traceback_fast = on; }
void nvb_debug_pair_extra_smem(int bytes) { nvb::g_pair_extra_smem = bytes > 0 ? bytes : 0; }
void nvb_debug_pair_format(int on) { nvb::g_pair_fmt_ok = on != 0; }
int nvb_debug_gotoh_last_route(int* packed, uint32_t* n_int32)
{
    if (!packed || !n_int32) return NVB_E_INVALID;
    *packed = g_route_packed;
    *n_int32 = 0u;
    if (!g_route_packed) return NVB_OK;
    NVB_CUDA_TRY(cudaDeviceSynchronize());
    NVB_CUDA_TRY(cudaMemcpy(n_int32, g_route_todo_count, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return NVB_OK;
}

} // extern "C"
