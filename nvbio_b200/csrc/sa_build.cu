// sa_build.cu -- suffix sorting / BWT / sampled-SA construction on the device.
//
// nvbio builds its test indices with a serial host SA-IS (contrib/sais.h via nvbio/fmindex/bwt.h:38-63)
// and real ones offline with nvBWT.  Here the index of a synthetic multi-gigabase genome is built in
// HBM in seconds: an 80 GB part lets us radix-sort all n suffixes of a genome up to ~1.9 Gbp (~40 bytes per
// base at the peak) by their first 32 symbols (one 64-bit key each) in one shot, then resolve the (for random genomes: almost non-existent) ties by prefix
// doubling over the tied groups only.
//
// Conventions reproduced (nvbio/fmindex/bwt.h:51-63, ssa_inl.h:262-277, io/fmindex/fmindex_impl.cu:244):
//   SA has n+1 rows, row 0 is the empty suffix `$` (SA[0]=n); BWT row r holds T[SA[r]-1] and the `$` row
//   (primary = row with SA=0) is dropped from the stored BWT; ssa[r/16] = SA[r] for r%16==0, ssa[0]=-1.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

namespace nvb {

// 32 symbols (64 bits) of a 2-bit big-endian stream starting at symbol i; symbols >= n read as 0
__device__ __forceinline__ uint64_t prefix32(const uint32_t* __restrict__ text, uint64_t n, uint64_t n_words, uint64_t i)
{
    const uint64_t w = i >> 4;
    const uint32_t sh = 2u * (uint32_t)(i & 15u);
    const uint64_t w0 = (w     < n_words) ? text[w]     : 0u;
    const uint64_t w1 = (w + 1 < n_words) ? text[w + 1] : 0u;
    const uint64_t w2 = (w + 2 < n_words) ? text[w + 2] : 0u;
    uint64_t hi = (w0 << 32) | w1;                 // symbols 16w .. 16w+31
    uint64_t key = sh ? ((hi << sh) | (w2 >> (32u - sh))) : hi;
    const uint64_t left = n - i;                   // symbols that exist
    if (left < 32) key &= ~((~0ull) >> (2u * (uint32_t)left));     // left >= 1
    return key;
}

__global__ void __launch_bounds__(256)
sa_init_kernel(const uint32_t* __restrict__ text, uint64_t n, uint64_t n_words, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    const uint64_t i = n - 1 - k;                  // descending start order: a stable sort then puts the
    keys[k] = prefix32(text, n, n_words, i);       // shorter of two equal-key suffixes first
    vals[k] = (uint32_t)i;
}

// head[k] = 1 when sorted position k starts a new group of (so far) indistinguishable suffixes.
// A suffix with <= 32 symbols left is fully compared by its key + the stable order -> always a singleton.
__global__ void __launch_bounds__(256)
sa_flag_heads_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t n, uint8_t* __restrict__ head)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    bool h = true;
    if (k > 0) {
        const bool short_k = (n - vals[k])     <= 32;
        const bool short_p = (n - vals[k - 1]) <= 32;
        h = short_k || short_p || (keys[k] != keys[k - 1]);
    }
    head[k] = h ? 1 : 0;
}

// unresolved[k] = 1 when k belongs to a group of size >= 2
__global__ void __launch_bounds__(256)
sa_flag_unresolved_kernel(const uint8_t* __restrict__ head, uint64_t n, uint8_t* __restrict__ unres)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    const bool next_head = (k + 1 >= n) || head[k + 1];
    unres[k] = (head[k] && next_head) ? 0 : 1;
}

struct MaxOp { __host__ __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; } };

// headpos[k] = head[k] ? k : 0  -> inclusive max-scan gives every position its group head
__global__ void __launch_bounds__(256)
sa_headpos_kernel(const uint8_t* __restrict__ head, uint64_t n, uint32_t* __restrict__ headpos)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    headpos[k] = head[k] ? (uint32_t)k : 0u;
}

// rank[SA[k]] = group head of k, +1 (rank 0 is the empty suffix)
__global__ void __launch_bounds__(256)
sa_write_rank_kernel(const uint32_t* __restrict__ vals, const uint32_t* __restrict__ ghead, uint64_t n, uint32_t* __restrict__ rank)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    rank[vals[k]] = ghead[k] + 1u;
}

// for the compacted list of unresolved sorted positions: key = (group head << 32) | rank[SA + h]
__global__ void __launch_bounds__(256)
sa_doubling_keys_kernel(const uint32_t* __restrict__ pos, uint32_t m, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ ghead,
                        const uint32_t* __restrict__ rank, uint64_t n, uint64_t h, uint64_t* __restrict__ keys, uint32_t* __restrict__ sfx)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= m) return;
    const uint32_t k = pos[t];
    const uint32_t i = vals[k];
    const uint64_t p = (uint64_t)i + h;
    const uint32_t r2 = (p < n) ? rank[p] : 0u;
    keys[t] = ((uint64_t)ghead[k] << 32) | r2;
    sfx[t] = i;
}

// scatter the re-sorted suffixes back into their (unchanged) set of positions and refresh the head flags
__global__ void __launch_bounds__(256)
sa_doubling_scatter_kernel(const uint32_t* __restrict__ pos, uint32_t m, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ sfx,
                           uint32_t* __restrict__ vals, uint8_t* __restrict__ head)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= m) return;
    const uint32_t k = pos[t];
    vals[k] = sfx[t];
    // a new group starts where the (group, next-rank) key changes; positions that were heads stay heads
    if (t == 0 || keys[t] != keys[t - 1]) head[k] = 1;
}

__global__ void __launch_bounds__(256)
sa_find_primary_kernel(const uint32_t* __restrict__ vals, uint64_t n, uint32_t* __restrict__ primary)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= n) return;
    if (vals[k] == 0u) *primary = (uint32_t)(k + 1);       // row index = sorted position + 1 (row 0 is `$`)
}

__device__ __forceinline__ uint32_t text_sym(const uint32_t* __restrict__ text, uint64_t i)
{
    return (text[i >> 4] >> (30u - 2u * (uint32_t)(i & 15u))) & 3u;
}

// one thread per output BWT word (16 symbols)
__global__ void __launch_bounds__(256)
sa_emit_bwt_kernel(const uint32_t* __restrict__ text, const uint32_t* __restrict__ vals, uint64_t n, const uint32_t* __restrict__ primary_p,
                   uint32_t n_out_words, uint32_t* __restrict__ bwt)
{
    const uint32_t w = blockIdx.x * 256 + threadIdx.x;
    if (w >= n_out_words) return;
    const uint64_t primary = *primary_p;
    uint32_t word = 0;
#pragma unroll
    for (uint32_t s = 0; s < 16; ++s) {
        const uint64_t o = (uint64_t)w * 16 + s;            // index in the stored BWT (primary row removed)
        uint32_t c = 0;
        if (o < n) {
            const uint64_t r = (o < primary) ? o : o + 1;    // SA row
            const uint64_t i = (r == 0) ? n : vals[r - 1];   // suffix start (never 0 here)
            c = text_sym(text, i - 1);
        }
        word |= c << (30u - 2u * s);
    }
    bwt[w] = word;
}

__global__ void __launch_bounds__(256)
sa_emit_ssa_kernel(const uint32_t* __restrict__ vals, uint64_t n, uint64_t n_items, uint32_t interval, uint32_t* __restrict__ ssa)
{
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n_items) return;
    ssa[t] = (t == 0) ? 0xFFFFFFFFu : vals[t * interval - 1];
}

__global__ void __launch_bounds__(256)
sa_emit_sa_kernel(const uint32_t* __restrict__ vals, uint64_t n, uint32_t* __restrict__ sa)
{
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r > n) return;
    sa[r] = (r == 0) ? (uint32_t)n : vals[r - 1];
}

static inline uint32_t grid_for(uint64_t n) { return (uint32_t)((n + 255) / 256); }

} // namespace nvb

using namespace nvb;

extern "C" int nvb_fm_build_bwt(const uint32_t* d_text, uint32_t n32, uint32_t* d_bwt, uint32_t* h_primary,
                                uint32_t* d_ssa, uint32_t sa_interval, uint32_t* d_sa,
                                void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!temp_bytes || !h_primary || n32 == 0 || n32 > NVB_FM_MAX_LENGTH || !d_text) return NVB_E_INVALID;
    if (sa_interval == 0) sa_interval = 16;
    if (sa_interval & (sa_interval - 1)) return NVB_E_INVALID;
    const uint64_t n = n32;
    const uint64_t n_words = (n + 15) / 16;
    cudaStream_t s = as_stream(stream);

    // ---- temp layout -------------------------------------------------------------------------
    TempCarver tc(d_temp);
    uint64_t* keysA = tc.take<uint64_t>(n);
    uint64_t* keysB = tc.take<uint64_t>(n);
    uint32_t* valsA = tc.take<uint32_t>(n);
    uint32_t* valsB = tc.take<uint32_t>(n);
    uint8_t*  head  = tc.take<uint8_t>(n);
    uint8_t*  unres = tc.take<uint8_t>(n);
    uint32_t* d_scalars = tc.take<uint32_t>(8);             // [0] primary, [1] #unresolved
    size_t sort_bytes = 0, scan_bytes = 0, sel_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keysA, keysB, valsA, valsB, (int64_t)n, 0, 64, s));
    NVB_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, MaxOp(), (int64_t)n, s));
    NVB_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, sel_bytes, cub::CountingInputIterator<uint32_t>(0), (uint8_t*)nullptr, (uint32_t*)nullptr,
                                            (uint32_t*)nullptr, (int64_t)n, s));
    size_t cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
    if (sel_bytes > cub_bytes) cub_bytes = sel_bytes;
    char* cub_tmp = tc.take<char>(cub_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (!d_bwt) return NVB_E_INVALID;

    // ---- 1. sort all suffixes by their first 32 symbols ----------------------------------------
    sa_init_kernel<<<grid_for(n), 256, 0, s>>>(d_text, n, n_words, keysA, valsA);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_bytes, keysA, keysB, valsA, valsB, (int64_t)n, 0, 64, s));
    uint64_t* keys = keysB; uint32_t* vals = valsB;         // sorted
    sa_flag_heads_kernel<<<grid_for(n), 256, 0, s>>>(keys, vals, n, head);
    NVB_LAUNCH_CHECK();

    // ---- 2. prefix doubling over the tied groups ---------------------------------------------------
    // buffers reused from here on: keysA (u64 n) -> doubling keys in/out halves; valsA (u32 n) -> ghead
    uint32_t* ghead = valsA;
    uint32_t* rank  = (uint32_t*)keysA;                     // n u32
    uint32_t* pos   = (uint32_t*)keysA + n;                 // n u32 (second half of keysA)
    for (uint64_t h = 32; ; h *= 2) {
        sa_flag_unresolved_kernel<<<grid_for(n), 256, 0, s>>>(head, n, unres);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceSelect::Flagged(cub_tmp, sel_bytes, cub::CountingInputIterator<uint32_t>(0), unres, pos, d_scalars + 1, (int64_t)n, s));
        uint32_t m = 0;
        NVB_CUDA_TRY(cudaMemcpyAsync(&m, d_scalars + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        NVB_CUDA_TRY(cudaStreamSynchronize(s));
        if (m == 0) break;
        if (h >= 2 * n) return NVB_E_UNSUPPORTED;           // cannot happen: every suffix is unique by length n
        // group heads and ranks at depth h
        sa_headpos_kernel<<<grid_for(n), 256, 0, s>>>(head, n, ghead);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::InclusiveScan(cub_tmp, scan_bytes, ghead, ghead, MaxOp(), (int64_t)n, s));
        sa_write_rank_kernel<<<grid_for(n), 256, 0, s>>>(vals, ghead, n, rank);
        NVB_LAUNCH_CHECK();
        // sort the unresolved suffixes by (group, rank of the suffix h further on).  Scratch: m u64 keys in/out
        // + m u32 suffixes in/out = 24m bytes.  The dead 32-symbol keys (keysB, 8n bytes) hold it when
        // 3m <= n (always, for random genomes: m ~ 0); denser ties take a stream-ordered allocation.
        uint64_t *dk_in, *dk_out; uint32_t *sfx_in, *sfx_out;
        const bool own_alloc = ((uint64_t)m * 3 > n);
        if (own_alloc) {
            NVB_CUDA_TRY(cudaMallocAsync(&dk_in,   sizeof(uint64_t) * m, s));
            NVB_CUDA_TRY(cudaMallocAsync(&dk_out,  sizeof(uint64_t) * m, s));
            NVB_CUDA_TRY(cudaMallocAsync(&sfx_in,  sizeof(uint32_t) * m, s));
            NVB_CUDA_TRY(cudaMallocAsync(&sfx_out, sizeof(uint32_t) * m, s));
        } else {
            dk_in = keysB; dk_out = keysB + m;
            sfx_in = (uint32_t*)(keysB + 2 * (uint64_t)m); sfx_out = sfx_in + m;
        }
        sa_doubling_keys_kernel<<<grid_for(m), 256, 0, s>>>(pos, m, vals, ghead, rank, n, h, dk_in, sfx_in);
        NVB_LAUNCH_CHECK();
        size_t sb = sort_bytes;
        NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, sb, dk_in, dk_out, sfx_in, sfx_out, (int64_t)m, 0, 64, s));
        sa_doubling_scatter_kernel<<<grid_for(m), 256, 0, s>>>(pos, m, dk_out, sfx_out, vals, head);
        NVB_LAUNCH_CHECK();
        if (own_alloc) {
            NVB_CUDA_TRY(cudaFreeAsync(dk_in, s));  NVB_CUDA_TRY(cudaFreeAsync(dk_out, s));
            NVB_CUDA_TRY(cudaFreeAsync(sfx_in, s)); NVB_CUDA_TRY(cudaFreeAsync(sfx_out, s));
        }
    }

    // ---- 3. emit BWT / SSA / SA ------------------------------------------------------------------
    NVB_CUDA_TRY(cudaMemsetAsync(d_scalars, 0, sizeof(uint32_t), s));
    sa_find_primary_kernel<<<grid_for(n), 256, 0, s>>>(vals, n, d_scalars);
    NVB_LAUNCH_CHECK();
    const uint32_t n_out_words = (uint32_t)(((n + 63) / 64) * 4);
    sa_emit_bwt_kernel<<<grid_for(n_out_words), 256, 0, s>>>(d_text, vals, n, d_scalars, n_out_words, d_bwt);
    NVB_LAUNCH_CHECK();
    if (d_ssa) {
        const uint64_t n_items = (n + sa_interval) / sa_interval;
        sa_emit_ssa_kernel<<<grid_for(n_items), 256, 0, s>>>(vals, n, n_items, sa_interval, d_ssa);
        NVB_LAUNCH_CHECK();
    }
    if (d_sa) {
        sa_emit_sa_kernel<<<grid_for(n + 1), 256, 0, s>>>(vals, n, d_sa);
        NVB_LAUNCH_CHECK();
    }
    NVB_CUDA_TRY(cudaMemcpyAsync(h_primary, d_scalars, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    NVB_CUDA_TRY(cudaStreamSynchronize(s));
    return NVB_OK;
}
