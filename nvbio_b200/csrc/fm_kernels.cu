// fm_kernels.cu -- HP-A: FM-index rank / match / locate / FMIndexFilter and the occ-table builder.
//
// One query per thread, a whole SM's worth of independent 32-byte gathers in flight (the path is
// bound by random-sector HBM/L2 throughput, SURVEY.md 8d): each LF step issues one 256-bit load per
// distinct block (two when the range ends straddle blocks) and ~40 integer ops.
#include "fm_core.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

namespace nvb {

constexpr int FM_BLOCKDIM = 128;          // queries finish after different numbers of gathers: small CTAs hand their warp slots on sooner (see pipeline.cu, SEED_BLOCK)

__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_rank_kernel(const FmIndex f, const uint32_t* __restrict__ k, const uint8_t* __restrict__ c, uint32_t n,
               uint32_t* __restrict__ out)
{
    const uint32_t i = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (i >= n) return;
    out[i] = fm_rank1(f, k[i], c[i] & 3u);
}

__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_rank4_kernel(const FmIndex f, const uint32_t* __restrict__ k, uint32_t n, uint4* __restrict__ out)
{
    const uint32_t i = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (i >= n) return;
    out[i] = fm_rank4(f, k[i]);
}

template <int BITS, bool BE>
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_match_kernel(const FmIndex f, const StrSet q, uint32_t n, uint32_t flags, uint2* __restrict__ out)
{
    const uint32_t i = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (i >= n) return;
    uint32_t x, y;
    fm_match_one<BITS, BE>(f, q.words, str_off(q, i), str_len(q, i), flags, x, y);
    out[i] = make_uint2(x, y);
}

template <int BITS, bool BE>
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_match_approx_kernel(const FmIndex f, const StrSet q, uint32_t n, uint32_t flags, uint32_t exact_len, bool find_exact, uint32_t max_out,
                       uint2* __restrict__ out, uint32_t* __restrict__ counts, uint32_t* __restrict__ sums)
{
    const uint32_t i = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (i >= n) return;
    uint32_t sum = 0;
    const uint32_t cnt = fm_map_approx_one<BITS, BE>(f, q.words, str_off(q, i), str_len(q, i), exact_len, flags, find_exact,
                                                     out + (size_t)i * max_out, max_out, sum);
    counts[i] = cnt;
    if (sums) sums[i] = sum;
}

__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_locate_kernel(const FmIndex f, const uint32_t* __restrict__ rows, uint32_t n, uint32_t* __restrict__ out)
{
    const uint32_t i = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (i >= n) return;
    out[i] = fm_locate_one(f, rows[i]);
}

template <typename W, typename I>
__global__ void __launch_bounds__(FM_BLOCKDIM)
dict_rank_kernel(const W* __restrict__ text, const I* __restrict__ occ, uint32_t K, const I* __restrict__ idx, const uint8_t* __restrict__ c, uint32_t n,
                 I* __restrict__ out, int all4)
{
    const uint32_t t = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (t >= n) return;
    if (all4) { for (uint32_t s = 0; s < 4u; ++s) out[4u * (size_t)t + s] = dict_rank<W, I>(text, occ, K, idx[t], s); }
    else out[t] = dict_rank<W, I>(text, occ, K, idx[t], c[t] & 3u);
}

// generic build_occurrence_table<2,K> (rank_dictionary_inl.h:42-77): per-block symbol counts, then their exclusive scan
template <typename W, typename I>
__global__ void __launch_bounds__(256)
dict_block_counts_kernel(const W* __restrict__ text, uint64_t n_symbols, uint32_t K, uint64_t n_blocks, uint64_t lane_len, I* __restrict__ counts /* [4][n_blocks + 1] */)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k > n_blocks) return;
    I cnt[4] = { 0, 0, 0, 0 };
    if (k < n_blocks) {
        constexpr uint32_t SPW = dict_word<W>::SPW;
        const uint64_t first = k * K;
        const uint64_t valid = (n_symbols - first) < K ? (n_symbols - first) : K;
        for (uint32_t j = 0; j * SPW < valid; ++j) {
            const uint32_t keep = (valid - (uint64_t)j * SPW) < SPW ? (uint32_t)(valid - (uint64_t)j * SPW) : SPW;
            const W w = text[k * (K / SPW) + j];
            for (uint32_t s = 0; s < 4u; ++s) cnt[s] += word_rank<W>(w, s, keep);
        }
    }
    for (uint32_t s = 0; s < 4u; ++s) counts[s * lane_len + k] = cnt[s];
}
template <typename I>
__global__ void __launch_bounds__(256)
dict_interleave_occ_kernel(const I* __restrict__ scan, uint64_t n_blocks, uint64_t lane_len, I* __restrict__ occ)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n_blocks) return;
    for (uint32_t c = 0; c < 4u; ++c) occ[4u * k + c] = scan[c * lane_len + k];
}

// one level of the k-mer table: entry v of level t-1 (the range of a (t-1)-mer w) fans out to the four
// t-mers c.w (c prepended = consumed next by the backward search).  The c=0 child overwrites its own parent.
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_ktab_level_kernel(const FmIndex f, uint2* __restrict__ tab, uint32_t prev_entries)
{
    const uint32_t v = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (v >= prev_entries) return;
    const uint2 r = tab[v];
#pragma unroll
    for (int c = 3; c >= 0; --c) {
        uint32_t x = r.x, y = r.y;
        if (x <= y) fm_step(f, (uint32_t)c, x, y);        // an empty range stays as it is (match() stops there)
        tab[(uint32_t)c * prev_entries + v] = make_uint2(x, y);
    }
}

// the same with 16-byte entries {x, y, -, -} (STRIDE 1) or the first half of 32-byte ones (STRIDE 2: the other half is filled by
// fm_ktab32_fill_kernel), and the pass that fills the SA values into the one- and two-row 16-byte ones
template <uint32_t STRIDE>
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_ktab16_level_kernel(const FmIndex f, uint4* __restrict__ tab, uint32_t prev_entries)
{
    const uint32_t v = blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (v >= prev_entries) return;
    const uint4 r = tab[(size_t)v * STRIDE];
#pragma unroll
    for (int c = 3; c >= 0; --c) {
        uint32_t x = r.x, y = r.y;
        if (x <= y) fm_step(f, (uint32_t)c, x, y);
        tab[((size_t)c * prev_entries + v) * STRIDE] = make_uint4(x, y, 0u, 0u);
    }
}
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_ktab16_locate_kernel(const FmIndex f, uint4* __restrict__ tab, uint64_t entries)
{
    const uint64_t v = (uint64_t)blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (v >= entries) return;
    const uint4 e = tab[v];
    // full suffix array (checked by the caller): SA[x] (0xFFFFFFFF for the `$` row) for one-row ranges, SA[x] and SA[y] for two-row ones
    if (e.x == e.y)           tab[v].z = f.ssa[e.x];
    else if (e.y == e.x + 1u) { tab[v].z = f.ssa[e.x]; tab[v].w = f.ssa[e.y]; }
}

// one-row entries of a located table: .w = the (up to) 16 text symbols before SA[x], symbol SA[x]-1 in the lowest two bits;
// two-row entries (index with fewer than 0xC0000000 rows): .y = marker | the 7 symbols before SA[x] | those before SA[x+1] << 14
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_ktab16_context_kernel(const uint32_t* __restrict__ text, uint4* __restrict__ tab, uint64_t entries, uint32_t n_rows)
{
    const uint64_t v = (uint64_t)blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (v >= entries) return;
    const uint4 e = tab[v];
    if (e.x == e.y) tab[v].w = text_before(text, e.z, 16u);
    else if (e.y == e.x + 1u && n_rows < KTAB_TWO_ROW_MARK)
        tab[v].y = KTAB_TWO_ROW_MARK | text_before(text, e.z, 7u) | (text_before(text, e.w, 7u) << 14);
}

// the per-row array: rows[r] = {SA[r], the 16 text symbols before SA[r]} -- the suffix array read in order, the text gathered
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_rows_kernel(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ text, uint2* __restrict__ rows, uint64_t n_rows)
{
    const uint64_t r = (uint64_t)blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (r >= n_rows) return;
    const uint32_t pos = sa[r];
    rows[r] = make_uint2(pos, text_before(text, pos, 16u));
}

// every 32-byte entry of a wide table from its range {x, y} (left in its first half by the level kernels): ktab_wide_fill
__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_ktab32_fill_kernel(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ text, uint4* __restrict__ tab, uint64_t entries, uint32_t n)
{
    const uint64_t v = (uint64_t)blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (v >= entries) return;
    const uint4 e = tab[2u * v];
    uint32_t w[8];
    ktab_wide_fill(sa, text, n, e.x, e.y, w);
    tab[2u * v] = make_uint4(w[0], w[1], w[2], w[3]);
    tab[2u * v + 1u] = make_uint4(w[4], w[5], w[6], w[7]);
}

// range sizes as uint64 (filter_inl.h:36-42: 1 + y - x in uint32 arithmetic, widened)
struct RangeSize {
    __host__ __device__ __forceinline__ uint64_t operator()(const uint2& r) const { return (uint64_t)(uint32_t)(1u + r.y - r.x); }
};

// upper_bound over the inclusive slots (filter_inl.h:99-118)
__device__ __forceinline__ uint32_t upper_bound_u64(const uint64_t* __restrict__ a, uint32_t n, uint64_t v)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] <= v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(FM_BLOCKDIM)
fm_filter_locate_kernel(const FmIndex f, const uint2* __restrict__ ranges, const uint64_t* __restrict__ slots,
                        uint32_t n_queries, uint64_t begin, uint64_t count, uint2* __restrict__ hits)
{
    const uint64_t t = (uint64_t)blockIdx.x * FM_BLOCKDIM + threadIdx.x;
    if (t >= count) return;
    const uint64_t h = begin + t;
    const uint32_t slot = upper_bound_u64(slots, n_queries, h);
    if (slot >= n_queries) { hits[t] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu); return; }   // h beyond the last hit: no row to locate
    const uint64_t base = slot ? slots[slot - 1] : 0ull;
    const uint32_t row = ranges[slot].x + (uint32_t)(h - base);
    hits[t] = make_uint2(fm_locate_one(f, row), slot);
}

// ---------------------------------------------------------------------------------------------
// occ-table build + interleave on the device (the reference does this serially on the host,
// rank_dictionary_inl.h:42-77 + fmindex_impl.cu:263-331, and carries a TODO for a CUDA version)
// ---------------------------------------------------------------------------------------------
struct U4Add { __host__ __device__ __forceinline__ uint4 operator()(const uint4& a, const uint4& b) const {
    return make_uint4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); } };

__global__ void __launch_bounds__(256)
occ_block_counts_kernel(const uint32_t* __restrict__ bwt, uint32_t n, uint32_t n_blocks, uint4* __restrict__ counts)
{
    const uint32_t k = blockIdx.x * 256 + threadIdx.x;
    if (k >= n_blocks) return;
    const uint4 w = reinterpret_cast<const uint4*>(bwt)[k];
    const uint32_t ws[4] = { w.x, w.y, w.z, w.w };
    const uint32_t valid = (n - k * 64u) < 64u ? (n - k * 64u) : 64u;     // symbols of this block that exist
    uint32_t cnt[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int keep = (int)valid - 16 * q;
        const uint32_t kk = keep < 0 ? 0u : (keep > 16 ? 16u : (uint32_t)keep);
        const uint32_t mask = (uint32_t)(0xFFFFFFFF00000000ull >> (2 * kk));
#pragma unroll
        for (uint32_t c = 0; c < 4; ++c) cnt[c] += __popc(eq_flags(ws[q], c * 0x55555555u) & mask);
    }
    counts[k] = make_uint4(cnt[0], cnt[1], cnt[2], cnt[3]);
}

__global__ void __launch_bounds__(256)
occ_interleave_kernel(const uint32_t* __restrict__ bwt, const uint4* __restrict__ occ_excl, uint32_t n, uint32_t n_blocks,
                      FmBlock* __restrict__ out)
{
    const uint32_t k = blockIdx.x * 256 + threadIdx.x;
    if (k >= n_blocks) return;
    uint4 w = reinterpret_cast<const uint4*>(bwt)[k];
    // zero the padding symbols (positions >= n) so that the emitted index is deterministic
    const uint32_t valid = (n - k * 64u) < 64u ? (n - k * 64u) : 64u;
    uint32_t ws[4] = { w.x, w.y, w.z, w.w };
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int keep = (int)valid - 16 * q;
        const uint32_t kk = keep < 0 ? 0u : (keep > 16 ? 16u : (uint32_t)keep);
        ws[q] &= (uint32_t)(0xFFFFFFFF00000000ull >> (2 * kk));
    }
    const uint4 o = occ_excl[k];
    FmBlock b;
    b.bwt[0] = ws[0]; b.bwt[1] = ws[1]; b.bwt[2] = ws[2]; b.bwt[3] = ws[3];
    b.occ[0] = o.x; b.occ[1] = o.y; b.occ[2] = o.z; b.occ[3] = o.w;
    out[k] = b;
}

template <typename W, typename I>
static int dict_rank_launch(const void* text, const void* occ, uint32_t K, const void* idx, const uint8_t* c, uint32_t n, void* out, int all4, cudaStream_t s)
{
    dict_rank_kernel<W, I><<<(n + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, s>>>((const W*)text, (const I*)occ, K, (const I*)idx, c, n, (I*)out, all4);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}
template <typename W, typename I>
static int dict_build_occ_impl(const void* d_text, uint64_t n_symbols, uint32_t K, void* d_occ, uint64_t h_counts[4], void* d_temp, size_t* temp_bytes, cudaStream_t s)
{
    const uint64_t n_blocks = (n_symbols + K - 1) / K;
    const uint64_t lane_len = n_blocks + 1;                       // one extra entry per symbol: its total
    TempCarver tc(d_temp);
    I* counts = tc.take<I>(4 * lane_len);                         // lane-major: counts[c * lane_len + k]
    I* scan   = tc.take<I>(4 * lane_len);
    size_t scan_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, counts, scan, (long long)lane_len, s));
    char* scan_tmp = tc.take<char>(scan_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    const uint32_t grid = (uint32_t)((lane_len + 255) / 256);
    dict_block_counts_kernel<W, I><<<grid, 256, 0, s>>>((const W*)d_text, n_symbols, K, n_blocks, lane_len, counts);
    NVB_LAUNCH_CHECK();
    for (uint32_t c = 0; c < 4u; ++c)
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, counts + c * lane_len, scan + c * lane_len, (long long)lane_len, s));
    dict_interleave_occ_kernel<I><<<grid, 256, 0, s>>>(scan, n_blocks, lane_len, (I*)d_occ);
    NVB_LAUNCH_CHECK();
    if (h_counts) {
        for (int c = 0; c < 4; ++c) {
            I tot;
            NVB_CUDA_TRY(cudaMemcpyAsync(&tot, scan + c * lane_len + n_blocks, sizeof(I), cudaMemcpyDeviceToHost, s));
            NVB_CUDA_TRY(cudaStreamSynchronize(s));
            h_counts[c] = (uint64_t)tot;
        }
    }
    return NVB_OK;
}

} // namespace nvb

using namespace nvb;

extern "C" {

int nvb_version(void) { return NVB_VERSION; }

const char* nvb_error_string(int err)
{
    switch (err) {
    case NVB_OK:            return "success";
    case NVB_E_INVALID:     return "nvbio_b200: invalid argument";
    case NVB_E_TEMP_SIZE:   return "nvbio_b200: temp storage missing or too small";
    case NVB_E_CAPACITY:    return "nvbio_b200: output capacity exceeded";
    case NVB_E_UNSUPPORTED: return "nvbio_b200: unsupported configuration";
    }
    return err > 0 ? cudaGetErrorString((cudaError_t)err) : "nvbio_b200: unknown error";
}

int nvb_fm_build_ktab(const nvb_fm_index* fmi, uint32_t k, nvb_uint2* d_ktab, void* stream)
{
    if (!valid_fmindex(fmi) || k < 1 || k > 16 || !d_ktab) return NVB_E_INVALID;
    nvb_fm_index plain = *fmi; plain.d_ktab = nullptr; plain.ktab_k = 0; plain.ktab_located = 0;
    const FmIndex f = make_fmindex(&plain);
    cudaStream_t s = as_stream(stream);
    const uint2 root = make_uint2(0u, fmi->length);
    NVB_CUDA_TRY(cudaMemcpyAsync(d_ktab, &root, sizeof(uint2), cudaMemcpyHostToDevice, s));
    NVB_CUDA_TRY(cudaStreamSynchronize(s));              // `root` lives on this stack frame
    uint32_t prev = 1;
    for (uint32_t t = 1; t <= k; ++t, prev *= 4u) {
        fm_ktab_level_kernel<<<(prev + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, s>>>(f, (uint2*)d_ktab, prev);
        NVB_LAUNCH_CHECK();
    }
    return NVB_OK;
}

int nvb_fm_build_ktab_located(const nvb_fm_index* fmi, uint32_t k, void* d_ktab16, void* stream)
{
    if (!valid_fmindex(fmi) || k < 1 || k > 16 || !d_ktab16 || ((uintptr_t)d_ktab16 & 15u)) return NVB_E_INVALID;
    if (fmi->sa_interval != 1u || !fmi->d_ssa) return NVB_E_UNSUPPORTED;
    nvb_fm_index plain = *fmi; plain.d_ktab = nullptr; plain.ktab_k = 0; plain.ktab_located = 0;
    const FmIndex f = make_fmindex(&plain);
    cudaStream_t s = as_stream(stream);
    const uint4 root = make_uint4(0u, fmi->length, 0u, 0u);
    NVB_CUDA_TRY(cudaMemcpyAsync(d_ktab16, &root, sizeof(uint4), cudaMemcpyHostToDevice, s));
    NVB_CUDA_TRY(cudaStreamSynchronize(s));              // `root` lives on this stack frame
    uint32_t prev = 1;
    for (uint32_t t = 1; t <= k; ++t, prev *= 4u) {
        fm_ktab16_level_kernel<1><<<(prev + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, s>>>(f, (uint4*)d_ktab16, prev);
        NVB_LAUNCH_CHECK();
    }
    const uint64_t entries = 1ull << (2u * k);
    fm_ktab16_locate_kernel<<<(uint32_t)((entries + FM_BLOCKDIM - 1) / FM_BLOCKDIM), FM_BLOCKDIM, 0, s>>>(f, (uint4*)d_ktab16, entries);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_build_ktab_context(const nvb_fm_index* fmi, uint32_t k, const uint32_t* d_text, void* d_ktab16, void* stream)
{
    if (!d_text) return NVB_E_INVALID;
    const int r = nvb_fm_build_ktab_located(fmi, k, d_ktab16, stream);
    if (r != NVB_OK) return r;
    const uint64_t entries = 1ull << (2u * k);
    fm_ktab16_context_kernel<<<(uint32_t)((entries + FM_BLOCKDIM - 1) / FM_BLOCKDIM), FM_BLOCKDIM, 0, as_stream(stream)>>>(d_text, (uint4*)d_ktab16, entries, fmi->length);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_build_ktab_wide(const nvb_fm_index* fmi, uint32_t k, const uint32_t* d_text, void* d_ktab32, void* stream)
{
    if (!valid_fmindex(fmi) || k < 1 || k > 16 || !d_text || !d_ktab32 || ((uintptr_t)d_ktab32 & 31u)) return NVB_E_INVALID;
    if (fmi->sa_interval != 1u || !fmi->d_ssa) return NVB_E_UNSUPPORTED;
    nvb_fm_index plain = *fmi; plain.d_ktab = nullptr; plain.ktab_k = 0; plain.ktab_located = 0;
    const FmIndex f = make_fmindex(&plain);
    cudaStream_t s = as_stream(stream);
    const uint4 root = make_uint4(0u, fmi->length, 0u, 0u);
    NVB_CUDA_TRY(cudaMemcpyAsync(d_ktab32, &root, sizeof(uint4), cudaMemcpyHostToDevice, s));
    NVB_CUDA_TRY(cudaStreamSynchronize(s));              // `root` lives on this stack frame
    uint32_t prev = 1;
    for (uint32_t t = 1; t <= k; ++t, prev *= 4u) {
        fm_ktab16_level_kernel<2><<<(prev + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, s>>>(f, (uint4*)d_ktab32, prev);
        NVB_LAUNCH_CHECK();
    }
    const uint64_t entries = 1ull << (2u * k);
    fm_ktab32_fill_kernel<<<(uint32_t)((entries + FM_BLOCKDIM - 1) / FM_BLOCKDIM), FM_BLOCKDIM, 0, s>>>(fmi->d_ssa, d_text, (uint4*)d_ktab32, entries, fmi->length);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_build_rows(const nvb_fm_index* fmi, const uint32_t* d_text, nvb_uint2* d_rows, void* stream)
{
    if (!fmi || !fmi->d_bwt_occ || !d_text || !d_rows || ((uintptr_t)d_rows & 7u)) return NVB_E_INVALID;
    if (fmi->sa_interval != 1u || !fmi->d_ssa) return NVB_E_UNSUPPORTED;
    const uint64_t n_rows = (uint64_t)fmi->length + 1u;
    fm_rows_kernel<<<(uint32_t)((n_rows + FM_BLOCKDIM - 1) / FM_BLOCKDIM), FM_BLOCKDIM, 0, as_stream(stream)>>>(fmi->d_ssa, d_text, (uint2*)d_rows, n_rows);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_rank(const nvb_fm_index* fmi, const uint32_t* d_k, const uint8_t* d_c, uint32_t n,
                uint32_t* d_out, void* stream)
{
    if (!valid_fmindex(fmi) || (n && (!d_k || !d_c || !d_out))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    fm_rank_kernel<<<(n + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, as_stream(stream)>>>(make_fmindex(fmi), d_k, d_c, n, d_out);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_rank4(const nvb_fm_index* fmi, const uint32_t* d_k, uint32_t n, uint32_t* d_out4, void* stream)
{
    if (!valid_fmindex(fmi) || (n && (!d_k || !d_out4))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    fm_rank4_kernel<<<(n + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, as_stream(stream)>>>(make_fmindex(fmi), d_k, n, (uint4*)d_out4);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_match(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                 nvb_uint2* d_ranges, void* stream)
{
    if (!valid_fmindex(fmi) || !valid_strset(queries) || (n && !d_ranges)) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    const FmIndex f = make_fmindex(fmi);
    const StrSet q = make_strset(queries);
    const uint32_t grid = (n + FM_BLOCKDIM - 1) / FM_BLOCKDIM;
#define CALL(B, E) fm_match_kernel<B, E><<<grid, FM_BLOCKDIM, 0, as_stream(stream)>>>(f, q, n, flags, (uint2*)d_ranges)
    NVB_DISPATCH_STREAM(q.bits, q.big_endian, CALL);
#undef CALL
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_match_approx(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                        uint32_t exact_len, int find_exact, uint32_t max_out,
                        nvb_uint2* d_ranges, uint32_t* d_counts, uint32_t* d_range_sums, void* stream)
{
    if (!valid_fmindex(fmi) || !valid_strset(queries) || max_out == 0 || (n && (!d_ranges || !d_counts))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    nvb_fm_index plain = *fmi; plain.d_ktab = nullptr; plain.ktab_k = 0;      // ranges start mid-seed: no table look-up here
    const FmIndex f = make_fmindex(&plain);
    const StrSet q = make_strset(queries);
    const uint32_t grid = (n + FM_BLOCKDIM - 1) / FM_BLOCKDIM;
#define CALL(B, E) fm_match_approx_kernel<B, E><<<grid, FM_BLOCKDIM, 0, as_stream(stream)>>>(f, q, n, flags, exact_len, find_exact != 0, max_out, \
                                                                                           (uint2*)d_ranges, d_counts, d_range_sums)
    NVB_DISPATCH_STREAM(q.bits, q.big_endian, CALL);
#undef CALL
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_locate(const nvb_fm_index* fmi, const uint32_t* d_rows, uint32_t n, uint32_t* d_pos, void* stream)
{
    if (!valid_fmindex(fmi) || !fmi->d_ssa || (n && (!d_rows || !d_pos))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    fm_locate_kernel<<<(n + FM_BLOCKDIM - 1) / FM_BLOCKDIM, FM_BLOCKDIM, 0, as_stream(stream)>>>(make_fmindex(fmi), d_rows, n, d_pos);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

int nvb_fm_filter_rank(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                       nvb_uint2* d_ranges, uint64_t* d_slots, uint64_t* h_n_hits,
                       void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!temp_bytes || (n && (!d_ranges || !d_slots))) return NVB_E_INVALID;
    if (h_n_hits) *h_n_hits = 0;
    if (n == 0) { *temp_bytes = 0; return NVB_OK; }
    cub::TransformInputIterator<uint64_t, RangeSize, const uint2*> sizes((const uint2*)d_ranges, RangeSize());
    size_t need = 0;
    NVB_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, need, sizes, d_slots, (int)n, as_stream(stream)));
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    const int r = nvb_fm_match(fmi, queries, n, flags, d_ranges, stream);
    if (r != NVB_OK) return r;
    NVB_CUDA_TRY(cub::DeviceScan::InclusiveSum(d_temp, need, sizes, d_slots, (int)n, as_stream(stream)));
    if (h_n_hits) {
        NVB_CUDA_TRY(cudaMemcpyAsync(h_n_hits, d_slots + (n - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, as_stream(stream)));
        NVB_CUDA_TRY(cudaStreamSynchronize(as_stream(stream)));
    }
    return NVB_OK;
}

int nvb_fm_filter_locate(const nvb_fm_index* fmi, const nvb_uint2* d_ranges, const uint64_t* d_slots,
                         uint32_t n_queries, uint64_t begin, uint64_t end, nvb_uint2* d_hits, void* stream)
{
    if (!valid_fmindex(fmi) || !fmi->d_ssa || !d_ranges || !d_slots || end < begin) return NVB_E_INVALID;
    const uint64_t count = end - begin;
    if (count == 0) return NVB_OK;
    if (!d_hits || count > 0x7FFFFFFFull * FM_BLOCKDIM) return NVB_E_INVALID;
    const uint32_t grid = (uint32_t)((count + FM_BLOCKDIM - 1) / FM_BLOCKDIM);
    fm_filter_locate_kernel<<<grid, FM_BLOCKDIM, 0, as_stream(stream)>>>(make_fmindex(fmi), (const uint2*)d_ranges, d_slots,
                                                                        n_queries, begin, count, (uint2*)d_hits);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

static bool dict_args_ok(uint32_t word_bits, uint32_t index_bits, uint32_t K)
{
    if (!(word_bits == 32 || word_bits == 64) || !(index_bits == 32 || index_bits == 64)) return false;
    return K != 0 && K % (word_bits / 2u) == 0;
}
int nvb_dict_rank(const void* d_text, uint32_t word_bits, const void* d_occ, uint32_t index_bits, uint32_t K,
                  const void* d_i, const uint8_t* d_c, uint32_t n, void* d_out, void* stream)
{
    if (!dict_args_ok(word_bits, index_bits, K) || (n && (!d_text || !d_occ || !d_i || !d_c || !d_out))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    cudaStream_t s = as_stream(stream);
    if (word_bits == 32) return index_bits == 32 ? dict_rank_launch<uint32_t, uint32_t>(d_text, d_occ, K, d_i, d_c, n, d_out, 0, s)
                                                 : dict_rank_launch<uint32_t, uint64_t>(d_text, d_occ, K, d_i, d_c, n, d_out, 0, s);
    return index_bits == 32 ? dict_rank_launch<uint64_t, uint32_t>(d_text, d_occ, K, d_i, d_c, n, d_out, 0, s)
                            : dict_rank_launch<uint64_t, uint64_t>(d_text, d_occ, K, d_i, d_c, n, d_out, 0, s);
}
int nvb_dict_rank4(const void* d_text, uint32_t word_bits, const void* d_occ, uint32_t index_bits, uint32_t K,
                   const void* d_i, uint32_t n, void* d_out4, void* stream)
{
    if (!dict_args_ok(word_bits, index_bits, K) || (n && (!d_text || !d_occ || !d_i || !d_out4))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    cudaStream_t s = as_stream(stream);
    if (word_bits == 32) return index_bits == 32 ? dict_rank_launch<uint32_t, uint32_t>(d_text, d_occ, K, d_i, nullptr, n, d_out4, 1, s)
                                                 : dict_rank_launch<uint32_t, uint64_t>(d_text, d_occ, K, d_i, nullptr, n, d_out4, 1, s);
    return index_bits == 32 ? dict_rank_launch<uint64_t, uint32_t>(d_text, d_occ, K, d_i, nullptr, n, d_out4, 1, s)
                            : dict_rank_launch<uint64_t, uint64_t>(d_text, d_occ, K, d_i, nullptr, n, d_out4, 1, s);
}

int nvb_dict_build_occ(const void* d_text, uint32_t word_bits, uint64_t n_symbols, uint32_t K, uint32_t index_bits, void* d_occ, uint64_t h_counts[4],
                       void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!dict_args_ok(word_bits, index_bits, K) || !temp_bytes || (n_symbols && (!d_text || !d_occ))) return NVB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    if (word_bits == 32) return index_bits == 32 ? dict_build_occ_impl<uint32_t, uint32_t>(d_text, n_symbols, K, d_occ, h_counts, d_temp, temp_bytes, s)
                                                 : dict_build_occ_impl<uint32_t, uint64_t>(d_text, n_symbols, K, d_occ, h_counts, d_temp, temp_bytes, s);
    return index_bits == 32 ? dict_build_occ_impl<uint64_t, uint32_t>(d_text, n_symbols, K, d_occ, h_counts, d_temp, temp_bytes, s)
                            : dict_build_occ_impl<uint64_t, uint64_t>(d_text, n_symbols, K, d_occ, h_counts, d_temp, temp_bytes, s);
}

int nvb_fm_build_occ(const uint32_t* d_bwt, uint32_t n, void* d_bwt_occ, uint32_t h_L2[5],
                     void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!temp_bytes || !h_L2 || n > NVB_FM_MAX_LENGTH || (n && (!d_bwt || !d_bwt_occ))) return NVB_E_INVALID;
    const uint32_t n_blocks = (uint32_t)(((uint64_t)n + 63u) / 64u);     // n + 63 wraps a uint32 from n = 2^32 - 63 on
    TempCarver tc(d_temp);
    uint4* counts = tc.take<uint4>(n_blocks + 1);
    uint4* excl   = tc.take<uint4>(n_blocks + 1);
    size_t scan_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, counts, excl, U4Add(), make_uint4(0, 0, 0, 0), (int)(n_blocks + 1), as_stream(stream)));
    char* scan_tmp = tc.take<char>(scan_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    cudaStream_t s = as_stream(stream);
    // counts[n_blocks] = 0 so that excl[n_blocks] = totals
    NVB_CUDA_TRY(cudaMemsetAsync(counts + n_blocks, 0, sizeof(uint4), s));
    if (n_blocks) {
        occ_block_counts_kernel<<<(n_blocks + 255) / 256, 256, 0, s>>>(d_bwt, n, n_blocks, counts);
        NVB_LAUNCH_CHECK();
    }
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveScan(scan_tmp, scan_bytes, counts, excl, U4Add(), make_uint4(0, 0, 0, 0), (int)(n_blocks + 1), s));
    if (n_blocks) {
        occ_interleave_kernel<<<(n_blocks + 255) / 256, 256, 0, s>>>(d_bwt, excl, n, n_blocks, (FmBlock*)d_bwt_occ);
        NVB_LAUNCH_CHECK();
    }
    uint4 tot;
    NVB_CUDA_TRY(cudaMemcpyAsync(&tot, excl + n_blocks, sizeof(uint4), cudaMemcpyDeviceToHost, s));
    NVB_CUDA_TRY(cudaStreamSynchronize(s));
    h_L2[0] = 0; h_L2[1] = tot.x; h_L2[2] = tot.x + tot.y; h_L2[3] = tot.x + tot.y + tot.z; h_L2[4] = tot.x + tot.y + tot.z + tot.w;
    return NVB_OK;
}

} // extern "C"
