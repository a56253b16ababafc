// bgzf.cu -- nvb_bgzf_compress: BGZF members (a dynamic-Huffman or stored deflate block each) of 0xFF00-byte input blocks in device
// memory.  Three steps:
//   bgzf_compress_kernel  a resident grid, one CTA per block at a time, everything of the block in shared memory (see BgzfSmem):
//                         stage the input with 16-byte loads; CRC-32 per 128-byte chunk, combined by shifts; match finding in chunks of
//                         512 positions against a hash table that only earlier chunks have written (atomicMax of the position, so the
//                         table and the matches do not depend on timing); the greedy parse by per-segment walks that are redone until
//                         every segment starts where the previous one ends; histograms; package-merge code lengths (one thread per
//                         alphabet); the header (one thread); a block scan of the tokens' bit counts; the tokens ORed into the member
//                         in shared memory, or a stored block when that is not larger; the member to its 64 KiB temp slot;
//   bgzf_scan_kernel      one CTA: the exclusive scan of the member sizes into d_block_offsets (a few thousand members per call; no
//                         temp of its own, so the size query needs no device);
//   bgzf_copy_kernel      each member from its slot to d_out through a shared-memory span laid out like the output modulo 16, stored
//                         with aligned 16-byte stores (bytes only at the head and tail), as bam_write_kernel does.
// The byte count is a host value (nvb_bgzf_compress) or lives in device memory beside a host upper bound (bgzf_compress_device_count,
// which the BAM pipeline runs on nvb_bam_records' total so that no batch waits for it on the host).  The bound sizes the grids and the
// temp; each kernel reads the real count itself (bgzf_count): the resident grid strides over the blocks that exist, the scan repeats the
// total past them, the copy stops at them.  With a host count both are the same number, so there is one code path.
#include <cub/cub.cuh>
#include "bgzf_core.cuh"

namespace nvb {

constexpr uint32_t BGZF_THREADS = 512u;               // also the match finder's chunk of positions
constexpr uint32_t BGZF_SEG = 128u;                   // positions per thread in the parse, the CRC and the token passes
constexpr uint32_t BGZF_BITMAP = 2048u;               // words of a per-position bitmap (65,536 positions)
constexpr uint32_t BGZF_COPY_THREADS = 256u;
constexpr uint32_t BGZF_SCAN_THREADS = 256u;
static_assert(BGZF_THREADS * BGZF_SEG >= BGZF_BLOCK, "one segment per thread covers a block");
static_assert(BGZF_SEG % 32u == 0u && BGZF_THREADS % 32u == 0u, "segments and chunks are whole bitmap words");

struct BgzfSmem {
    uint8_t  in[BGZF_BLOCK + 16u];                    // the block, zero padded for 4-byte loads
    uint8_t  mlen[BGZF_BLOCK];                        // match length - 3 where mbit is set
    union {
        uint32_t hash[1u << BGZF_HASH_BITS];          // match finding: position + 1 of the latest inserted position per hash
        struct { BgzfPm lit, dist; } pm;              // code construction
        uint32_t out[BGZF_SLOT / 4u];                 // the member
    } u;
    uint32_t mbit[BGZF_BITMAP];                       // position has a match
    uint32_t tok[BGZF_BITMAP];                        // position starts a token of the parse
    uint32_t crc_table[256];
    uint32_t hlit[BGZF_NLIT], hdist[BGZF_NDIST];
    BgzfCodes codes;
    uint32_t exits[BGZF_THREADS];                     // first token start at or past the end of each segment
    uint32_t crc_warp[BGZF_THREADS / 32u];
    uint32_t bits;                                    // bits of all tokens
    typename cub::BlockScan<uint32_t, BGZF_THREADS>::TempStorage scan;
};
static_assert(sizeof(BgzfSmem) <= 227u * 1024u, "one CTA per SM: an H100 CTA gets at most 227 KB of shared memory");

// the byte count: the device value when there is one (never above the host bound), else the host value
__device__ __forceinline__ uint64_t bgzf_count(const uint64_t n_bytes, const uint64_t* __restrict__ d_n_bytes)
{
    return d_n_bytes ? min(*d_n_bytes, n_bytes) : n_bytes;
}
__device__ __forceinline__ uint32_t bgzf_blocks(const uint64_t n) { return (uint32_t)(n / BGZF_BLOCK + (n % BGZF_BLOCK != 0u)); }

// the parse walk of segment [s0, s1) from entry g: marks its token starts and returns the first position at or past s1
__device__ __forceinline__ uint32_t bgzf_walk(BgzfSmem& S, const BgzfParse& v, uint32_t s0, uint32_t s1, uint32_t g)
{
    uint32_t* tok = S.tok + s0 / 32u;
#pragma unroll
    for (uint32_t k = 0; k < BGZF_SEG / 32u; ++k) tok[k] = 0u;
    uint32_t p = g;
    for (; p < s1; p += token_advance(v, p)) tok[(p - s0) >> 5] |= 1u << (p & 31u);
    return p;
}

__global__ void __launch_bounds__(BGZF_THREADS, 1)
bgzf_compress_kernel(const uint8_t* __restrict__ d_in, const uint64_t n_bound, const uint64_t* __restrict__ d_n_bytes, uint8_t* __restrict__ slots,
                     uint16_t* __restrict__ dist_scratch, uint64_t* __restrict__ sizes)
{
    const uint64_t n_bytes = bgzf_count(n_bound, d_n_bytes);
    const uint32_t n_blocks = bgzf_blocks(n_bytes);
    extern __shared__ __align__(16) uint8_t smem_raw[];
    BgzfSmem& S = *reinterpret_cast<BgzfSmem*>(smem_raw);
    const uint32_t t = threadIdx.x, lane = t & 31u;
    uint16_t* dist = dist_scratch + (size_t)blockIdx.x * BGZF_BLOCK;
    const BgzfParse v{ S.in, S.mlen, S.mbit, dist };
    if (t < 256u) S.crc_table[t] = crc32_table_entry(t);

    for (uint32_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const uint64_t base = (uint64_t)blk * BGZF_BLOCK;
        const uint32_t n = (uint32_t)(n_bytes - base < BGZF_BLOCK ? n_bytes - base : BGZF_BLOCK);
        const uint8_t* src = d_in + base;
        // stage; clear the table, the bitmaps and the histograms
        uint32_t i0 = 0u;
        if (((uintptr_t)src & 15u) == 0u) {
            i0 = n & ~15u;
            for (uint32_t i = 16u * t; i < i0; i += 16u * BGZF_THREADS) *(uint4*)(S.in + i) = __ldg((const uint4*)(src + i));
        }
        for (uint32_t i = i0 + t; i < n; i += BGZF_THREADS) S.in[i] = src[i];
        if (t < 16u) S.in[n + t] = 0u;
        for (uint32_t i = t; i < (1u << BGZF_HASH_BITS); i += BGZF_THREADS) S.u.hash[i] = 0u;
        for (uint32_t i = t; i < BGZF_BITMAP; i += BGZF_THREADS) S.mbit[i] = 0u;
        for (uint32_t i = t; i < BGZF_NLIT; i += BGZF_THREADS) S.hlit[i] = i == 256u ? 1u : 0u;
        if (t < BGZF_NDIST) S.hdist[t] = 0u;
        __syncthreads();

        // CRC-32: register of segment t from 0, shifted past the rest of the block; the XOR of all with the shifted initial register
        const uint32_t s0 = t * BGZF_SEG, s1 = min(n, s0 + BGZF_SEG);
        uint32_t crc = 0u;
        if (s0 < n) crc = crc32_shift(crc32_raw(S.crc_table, S.in + s0, s1 - s0, 0u), n - s1);
        if (t == 0u) crc ^= crc32_shift(0xFFFFFFFFu, n);
        crc = __reduce_xor_sync(0xFFFFFFFFu, crc);
        if (lane == 0u) S.crc_warp[t >> 5] = crc;

        // match finding: chunk c looks up the table as chunks < c left it, then inserts its positions
        for (uint32_t c0 = 0; c0 < n; c0 += BGZF_THREADS) {
            const uint32_t p = c0 + t;
            const bool hashable = p + 4u <= n;
            const uint32_t h = hashable ? bgzf_hash(S.in, p) : 0u;
            const uint32_t m = p < n ? find_match(S.in, n, p, hashable ? S.u.hash[h] : 0u) : 0u;
            if (m) { S.mlen[p] = (uint8_t)((m >> 16) - 3u); dist[p] = (uint16_t)(m & 0xFFFFu); }
            const uint32_t ball = __ballot_sync(0xFFFFFFFFu, m != 0u);
            if (lane == 0u) S.mbit[p >> 5] = ball;
            __syncthreads();
            if (hashable) atomicMax(S.u.hash + h, p + 1u);
            __syncthreads();
        }

        // greedy parse: walk every segment from its start, then redo the walks whose entry (the previous segment's exit) differs, until
        // none does; segment 0 starts at 0, so the fixed point is the greedy parse of the block
        uint32_t g = s0;
        S.exits[t] = bgzf_walk(S, v, s0, s1, g);
        __syncthreads();
        for (;;) {
            const uint32_t e = t ? S.exits[t - 1u] : 0u;
            __syncthreads();
            const bool redo = e != g;
            if (redo) { g = e; S.exits[t] = bgzf_walk(S, v, s0, s1, g); }
            if (!__syncthreads_or(redo)) break;
        }

        // histograms of the tokens
#pragma unroll 1
        for (uint32_t k = 0; k < BGZF_SEG / 32u; ++k)
            for (uint32_t b = S.tok[s0 / 32u + k]; b; b &= b - 1u) count_token(v, s0 + 32u * k + bgzf_ctz(b), S.hlit, S.hdist);
        __syncthreads();

        // code lengths: the used symbols of each alphabet ranked in parallel, then package-merge by one thread per alphabet
        if (t == 0u) bump_used(S.hlit, BGZF_NLIT);
        if (t == 32u) bump_used(S.hdist, BGZF_NDIST);
        __syncthreads();
        if (t < BGZF_NLIT && S.hlit[t]) {
            const uint32_t r = freq_rank(S.hlit, BGZF_NLIT, t);
            S.u.pm.lit.sym[r] = (uint16_t)t; S.u.pm.lit.w[r] = S.hlit[t];
        }
        if (t >= 384u && t < 384u + BGZF_NDIST && S.hdist[t - 384u]) {
            const uint32_t s = t - 384u, r = freq_rank(S.hdist, BGZF_NDIST, s);
            S.u.pm.dist.sym[r] = (uint16_t)s; S.u.pm.dist.w[r] = S.hdist[s];
        }
        const uint32_t m_lit = __syncthreads_count(t < BGZF_NLIT && S.hlit[t]);
        const uint32_t m_dist = __syncthreads_count(t < BGZF_NDIST && S.hdist[t]);
        if (t == 0u) package_merge(S.u.pm.lit, m_lit, BGZF_MAX_BITS, S.codes.lit_len);
        if (t == 32u) package_merge(S.u.pm.dist, m_dist, BGZF_MAX_BITS, S.codes.dist_len);
        if (t >= 64u && t < 64u + BGZF_NLIT && !S.hlit[t - 64u]) S.codes.lit_len[t - 64u] = 0u;
        if (t >= 384u && t < 384u + BGZF_NDIST && !S.hdist[t - 384u]) S.codes.dist_len[t - 384u] = 0u;
        __syncthreads();
        if (t == 0u) plan_header(S.codes, S.u.pm.lit);
        __syncthreads();

        // bit offsets of the segments' tokens; the member's size; dynamic or stored
        uint32_t my_bits = 0u;
#pragma unroll 1
        for (uint32_t k = 0; k < BGZF_SEG / 32u; ++k)
            for (uint32_t b = S.tok[s0 / 32u + k]; b; b &= b - 1u) my_bits += put_token(v, S.codes, s0 + 32u * k + bgzf_ctz(b), nullptr, 0u);
        uint32_t my_off;
        cub::BlockScan<uint32_t, BGZF_THREADS>(S.scan).ExclusiveSum(my_bits, my_off);
        if (t == BGZF_THREADS - 1u) S.bits = my_off + my_bits;
        for (uint32_t i = t; i < BGZF_SLOT / 4u; i += BGZF_THREADS) S.u.out[i] = 0u;
        __syncthreads();
        const uint32_t hb = S.codes.header_bits, total = hb + S.bits + S.codes.lit_len[256];
        const uint32_t dbytes = (total + 7u) / 8u;
        const bool stored = dbytes >= n + 5u;
        const uint32_t member = BGZF_HDR + (stored ? n + 5u : dbytes) + BGZF_FTR;
        uint8_t* out8 = reinterpret_cast<uint8_t*>(S.u.out);
        if (stored) {
            for (uint32_t i = t; i < n; i += BGZF_THREADS) out8[BGZF_HDR + 5u + i] = S.in[i];
        } else {
            const uint32_t pos0 = 8u * BGZF_HDR;
            if (t == 0u) write_header(S.u.out, pos0, S.codes);
            uint32_t pos = pos0 + hb + my_off;
#pragma unroll 1
            for (uint32_t k = 0; k < BGZF_SEG / 32u; ++k)
                for (uint32_t b = S.tok[s0 / 32u + k]; b; b &= b - 1u) pos += put_token(v, S.codes, s0 + 32u * k + bgzf_ctz(b), S.u.out, pos);
            if (t == BGZF_THREADS - 1u) put_bits(S.u.out, pos, S.codes.lit_code[256], S.codes.lit_len[256]);
        }
        __syncthreads();
        // framing bytes (after the bit stream's atomics: they share words with it)
        if (t < BGZF_HDR) out8[t] = member_header_byte(t, member);
        else if (t < BGZF_HDR + BGZF_FTR) {
            uint32_t c = 0u;
            for (uint32_t w = 0; w < BGZF_THREADS / 32u; ++w) c ^= S.crc_warp[w];
            out8[member - BGZF_FTR + (t - BGZF_HDR)] = member_footer_byte(t - BGZF_HDR, ~c, n);
        } else if (stored && t < BGZF_HDR + BGZF_FTR + 5u) out8[BGZF_HDR + (t - BGZF_HDR - BGZF_FTR)] = stored_header_byte(t - BGZF_HDR - BGZF_FTR, n);
        __syncthreads();
        uint4* slot = reinterpret_cast<uint4*>(slots + (size_t)blk * BGZF_SLOT);
        for (uint32_t i = t; i < (member + 15u) / 16u; i += BGZF_THREADS) slot[i] = reinterpret_cast<const uint4*>(S.u.out)[i];
        if (t == 0u) sizes[blk] = member;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BGZF_SCAN_THREADS)
bgzf_scan_kernel(const uint64_t* __restrict__ sizes, const uint64_t n_bound, const uint64_t* __restrict__ d_n_bytes, uint64_t* __restrict__ offsets)
{
    typedef cub::BlockScan<uint64_t, BGZF_SCAN_THREADS> Scan;
    __shared__ typename Scan::TempStorage ts;
    const uint32_t n_blocks = bgzf_blocks(bgzf_count(n_bound, d_n_bytes)), n_out = bgzf_blocks(n_bound);
    uint64_t carry = 0u;
    for (uint64_t b = 0; b <= n_out; b += BGZF_SCAN_THREADS) {     // n_out + 1 outputs: [n_blocks] is the total, repeated after it
        const uint64_t i = b + threadIdx.x;
        uint64_t y, sum;
        Scan(ts).ExclusiveSum(i < n_blocks ? sizes[i] : 0u, y, sum);
        if (i <= n_out) offsets[i] = carry + y;
        carry += sum;
        __syncthreads();
    }
}

// members whose end fits the capacity, from their slots to d_out
__global__ void __launch_bounds__(BGZF_COPY_THREADS)
bgzf_copy_kernel(const uint8_t* __restrict__ slots, const uint64_t* __restrict__ offsets, const uint64_t n_bound, const uint64_t* __restrict__ d_n_bytes,
                 uint8_t* __restrict__ out, const uint64_t capacity)
{
    extern __shared__ __align__(16) uint8_t stage[];                   // BGZF_SLOT + 16 bytes
    const uint32_t t = threadIdx.x;
    const uint32_t n_blocks = bgzf_blocks(bgzf_count(n_bound, d_n_bytes));
    for (uint32_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const uint64_t lo = offsets[blk], hi = offsets[blk + 1u];
        if (hi > capacity) return;                                     // so are all later members
        const uint32_t len = (uint32_t)(hi - lo);
        uint8_t* dst = out + lo;
        const uint32_t sh = (uint32_t)((uintptr_t)dst & 15u);          // member byte k at stage[sh + k]
        const uint4* src = reinterpret_cast<const uint4*>(slots + (size_t)blk * BGZF_SLOT);
        for (uint32_t i = t; i < (len + 15u) / 16u; i += BGZF_COPY_THREADS) {
            const uint4 x = src[i];
            const uint32_t w[4] = { x.x, x.y, x.z, x.w };
#pragma unroll
            for (uint32_t k = 0; k < 16u; ++k) stage[sh + 16u * i + k] = (uint8_t)(w[k >> 2] >> (8u * (k & 3u)));
        }
        __syncthreads();
        const uint32_t a0 = min(len, (16u - sh) & 15u);                // member bytes before the first aligned line
        const uint32_t a1 = a0 + ((len - a0) & ~15u);                  // ... and after the last
        for (uint32_t k = t; k < a0; k += BGZF_COPY_THREADS) dst[k] = stage[sh + k];
        for (uint32_t k = a0 + 16u * t; k < a1; k += 16u * BGZF_COPY_THREADS) *(uint4*)(dst + k) = *(const uint4*)(stage + sh + k);
        for (uint32_t k = a1 + t; k < len; k += BGZF_COPY_THREADS) dst[k] = stage[sh + k];
        __syncthreads();
    }
}

static uint32_t g_bgzf_grid = 0u;                                      // nvb_debug_bgzf_grid: 0 = one CTA per SM

int bgzf_compress_device_count(const uint8_t* d_in, uint64_t n_bytes, const uint64_t* d_n_bytes, const nvb_bgzf_out* out, void* d_temp,
                               size_t* temp_bytes, void* stream)
{
    if (!out || !temp_bytes || (!d_in && n_bytes) || !out->d_block_offsets || (!out->d_out && out->capacity)) return NVB_E_INVALID;
    const uint64_t nb = n_bytes / BGZF_BLOCK + (n_bytes % BGZF_BLOCK != 0u);
    if (nb >= (1ull << 32)) return NVB_E_INVALID;
    const cudaStream_t s = as_stream(stream);
    if (nb == 0u) {
        *temp_bytes = 0;
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_block_offsets, 0, sizeof(uint64_t), s));
        return NVB_OK;
    }
    const uint32_t grid = (uint32_t)std::min<uint64_t>(nb, g_bgzf_grid ? g_bgzf_grid : sm_count());
    TempCarver tc(nullptr);
    tc.take<uint8_t>(nb * BGZF_SLOT); tc.take<uint64_t>(nb); tc.take<uint16_t>((size_t)grid * BGZF_BLOCK);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    TempCarver tt(d_temp);
    uint8_t* slots = tt.take<uint8_t>(nb * BGZF_SLOT);
    uint64_t* sizes = tt.take<uint64_t>(nb);
    uint16_t* dist = tt.take<uint16_t>((size_t)grid * BGZF_BLOCK);

    const int smem = (int)sizeof(BgzfSmem), copy_smem = (int)(BGZF_SLOT + 16u);
    NVB_CUDA_TRY(cudaFuncSetAttribute(bgzf_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    NVB_CUDA_TRY(cudaFuncSetAttribute(bgzf_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, copy_smem));
    bgzf_compress_kernel<<<grid, BGZF_THREADS, smem, s>>>(d_in, n_bytes, d_n_bytes, slots, dist, sizes);
    NVB_LAUNCH_CHECK();
    bgzf_scan_kernel<<<1, BGZF_SCAN_THREADS, 0, s>>>(sizes, n_bytes, d_n_bytes, out->d_block_offsets);
    NVB_LAUNCH_CHECK();
    if (out->capacity == 0u) return NVB_OK;
    const uint32_t copy_grid = (uint32_t)std::min<uint64_t>(nb, 4u * (uint64_t)sm_count());
    bgzf_copy_kernel<<<copy_grid, BGZF_COPY_THREADS, copy_smem, s>>>(slots, out->d_block_offsets, n_bytes, d_n_bytes, out->d_out, out->capacity);
    return (int)cudaGetLastError();
}

} // namespace nvb

using namespace nvb;

extern "C" void nvb_debug_bgzf_grid(uint32_t ctas) { g_bgzf_grid = ctas; }

extern "C" int nvb_bgzf_compress(const uint8_t* d_in, uint64_t n_bytes, const nvb_bgzf_out* out, void* d_temp, size_t* temp_bytes, void* stream)
{
    return bgzf_compress_device_count(d_in, n_bytes, nullptr, out, d_temp, temp_bytes, stream);
}

extern "C" int nvb_debug_bgzf_compress_device_count(const uint8_t* d_in, const uint64_t* d_n_bytes, uint64_t max_bytes, const nvb_bgzf_out* out,
                                                    void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!d_n_bytes) return NVB_E_INVALID;
    return bgzf_compress_device_count(d_in, max_bytes, d_n_bytes, out, d_temp, temp_bytes, stream);
}
