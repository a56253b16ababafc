// bam_sort.cu -- coordinate sort of BAM records (nvb_bam_sort) and the BAI index of the sorted, BGZF-compressed records (nvb_bam_index),
// both on the device with no host round trip.  The rules are stated once, in include/nvbio_b200.h.
//
// nvb_bam_sort:
//   bam_sort_key_kernel     a thread per record: key = refID:pos (read bytewise, records start anywhere), value = its index;
//   a stable radix sort     of the 64-bit keys with 32-bit values (CUB);
//   bam_sort_size_kernel    the record sizes in sorted order, then an exclusive scan of them into d_offsets (CUB);
//   bam_gather_kernel       a CTA takes SORT_RUN consecutive OUTPUT records, copies them (a warp per record, aligned 16-byte loads inside the
//                           source record) into a shared-memory span laid out like the output modulo 16, and stores the span with aligned
//                           16-byte stores, as bam_write_kernel does.  A record larger than the span is copied directly.
// nvb_bam_index:
//   bai_record_kernel       a thread per record: refID, pos, CIGAR reference length, bin, the order / range checks, the mapped-end value of
//                           the linear index scan;  bai_head_kernel: run heads of equal (refID, bin), each refID's record range;
//   chunks                  an exclusive scan of the heads numbers the chunks, bai_chunk_kernel fills them ([start, end) virtual offsets);
//   five level passes       chunks sorted (stably, so by start inside a bin) by refID:bin; bai_level_kernel moves the chunks of a bin at
//                           level l to its parent when compress_binning would; a re-sort after each pass;
//   absorption              bai_absorb_kernel + a scan: a chunk that starts in the BGZF block where the previous one of its bin ends joins it;
//   sizing                  a scan of the bin heads, bai_ref_size_kernel per refID, a scan over refIDs;
//   writers                 bai_chunk_write_kernel (bins and chunks), bai_ref_write_kernel (BAI_REF_CTAS CTAs per refID: n_bin, the pseudo-bin,
//                           the linear index by two binary searches per window over the refID's prefix maximum of mapped ends).
#include <cub/cub.cuh>
#include "bam_core.cuh"

namespace nvb {

constexpr uint32_t SORT_RUN = 64u;                  // output records per CTA of the gather kernel
constexpr uint32_t SORT_STAGE = 32768u;             // bytes of its staging span
constexpr uint32_t SORT_THREADS = 256u;
constexpr uint64_t BAI_BLOCK = 0xFF00u;             // uncompressed bytes per BGZF member (nvb_bgzf_compress)
constexpr uint32_t BAI_META_BIN = 37450u;
constexpr uint32_t BAI_UNPLACED_BIN = 4680u;
constexpr uint32_t BAI_NO_REF = 0xFFFFFFFFu;
constexpr uint32_t BAI_REF_CTAS = 16u;              // CTAs per refID of the linear index writer

__device__ __forceinline__ uint32_t get32(const uint8_t* p)
{
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ void put64(uint8_t* p, uint64_t v) { put32(p, (uint32_t)v); put32(p + 4, (uint32_t)(v >> 32)); }

// refID:pos of the record at p with `len` bytes; bytes past the record read as 0xFF
__device__ __forceinline__ uint64_t sort_key(const uint8_t* p, uint64_t len)
{
    uint64_t k = 0u;
    for (uint32_t b = 0; b < 8u; ++b) {                                 // refID: bytes 4-7, the high word; pos: bytes 8-11
        const uint64_t v = 4u + b < len ? p[4u + b] : 0xFFu;
        k |= v << (b < 4u ? 32u + 8u * b : 8u * (b - 4u));
    }
    return k;
}

__global__ void __launch_bounds__(128)
bam_sort_key_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ off, const uint32_t n, uint64_t* __restrict__ keys,
                    uint32_t* __restrict__ idx)
{
    const uint32_t i = blockIdx.x * 128u + threadIdx.x;
    if (i >= n) return;
    const uint64_t s = off[i];
    keys[i] = sort_key(in + s, off[i + 1u] - s);
    idx[i] = i;
}

__global__ void __launch_bounds__(128)
bam_sort_size_kernel(const uint64_t* __restrict__ off, const uint32_t* __restrict__ order, const uint32_t n, uint64_t* __restrict__ sizes)
{
    const uint32_t j = blockIdx.x * 128u + threadIdx.x;
    if (j < n) { const uint32_t i = order[j]; sizes[j] = off[i + 1u] - off[i]; }
    else if (j == n) sizes[n] = 0u;                                       // the scan's extra element: d_offsets[n] = the total
}

// len bytes from global src to dst (shared or global), `lanes` threads from `lane`: whole aligned 16-byte lines of the source are loaded as
// such, the partial lines at either end byte by byte, so no load leaves the record
__device__ __forceinline__ void copy_record(uint8_t* dst, const uint8_t* src, const uint64_t len, const uint32_t lane, const uint32_t lanes)
{
    const uintptr_t a = (uintptr_t)src, z = a + len;
    for (uintptr_t line = (a & ~(uintptr_t)15u) + 16u * lane; line < z; line += 16u * lanes) {
        if (line >= a && line + 16u <= z) {
            const uint4 x = *reinterpret_cast<const uint4*>(line);
            const uint32_t w[4] = { x.x, x.y, x.z, x.w };
            uint8_t* d = dst + (line - a);
#pragma unroll
            for (uint32_t k = 0; k < 16u; ++k) d[k] = (uint8_t)(w[k >> 2] >> (8u * (k & 3u)));
        } else {
            for (uintptr_t p = line < a ? a : line; p < line + 16u && p < z; ++p) dst[p - a] = *reinterpret_cast<const uint8_t*>(p);
        }
    }
}

__global__ void __launch_bounds__(SORT_THREADS)
bam_gather_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ in_off, const uint32_t* __restrict__ order,
                  const uint64_t* __restrict__ out_off, const uint32_t n, uint8_t* __restrict__ out, const uint64_t capacity)
{
    __shared__ __align__(16) uint8_t stage[SORT_STAGE];
    __shared__ uint64_t so[SORT_RUN + 1u], si[SORT_RUN];
    const uint32_t r0 = blockIdx.x * SORT_RUN, r1 = min(n, r0 + SORT_RUN);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = threadIdx.x; i <= r1 - r0; i += SORT_THREADS) {
        so[i] = out_off[r0 + i];
        if (i < r1 - r0) si[i] = in_off[order[r0 + i]];
    }
    __syncthreads();
    // records that fit the capacity are a prefix: record k is stored when out_off[k + 1] <= capacity
    for (uint32_t r = r0; r < r1 && so[r + 1u - r0] <= capacity;) {
        const uint64_t base = so[r - r0] & ~(uint64_t)15u;
        uint32_t e = r + 1u;
        while (e < r1 && so[e + 1u - r0] <= capacity && so[e + 1u - r0] - base <= SORT_STAGE) ++e;
        if (so[e - r0] - base > SORT_STAGE) {                            // record r alone is larger than the span
            copy_record(out + so[r - r0], in + si[r - r0], so[r + 1u - r0] - so[r - r0], threadIdx.x, SORT_THREADS);
            r = e;
            continue;
        }
        for (uint32_t k = r + warp; k < e; k += SORT_THREADS / 32u)
            copy_record(stage + (so[k - r0] - base), in + si[k - r0], so[k + 1u - r0] - so[k - r0], lane, 32u);
        __syncthreads();
        // store [lo, hi): whole 16-byte lines from the span, the partial lines at either end byte by byte
        const uint64_t lo = so[r - r0], hi = so[e - r0];
        const uint64_t a0 = (lo + 15u) & ~(uint64_t)15u, a1 = hi & ~(uint64_t)15u;
        if (a0 >= a1) {
            for (uint64_t g = lo + threadIdx.x; g < hi; g += SORT_THREADS) out[g] = stage[g - base];
        } else {
            for (uint64_t g = lo + threadIdx.x; g < a0; g += SORT_THREADS) out[g] = stage[g - base];
            for (uint64_t g = a0 + 16u * threadIdx.x; g < a1; g += 16u * SORT_THREADS)
                *(uint4*)(out + g) = *(const uint4*)(stage + (g - base));
            for (uint64_t g = a1 + threadIdx.x; g < hi; g += SORT_THREADS) out[g] = stage[g - base];
        }
        __syncthreads();
        r = e;
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// BAI

struct BaiFile {
    const uint64_t* rec_off;      // [n + 1] uncompressed record offsets
    const uint64_t* blk_off;      // [n_blocks + 1] member offsets of the compressed records
    uint64_t header_bytes;        // compressed bytes before the first member
    uint32_t n;
    // the virtual offset htslib's reader reports at uncompressed byte u of the records: it moves to the next member as soon as it has
    // consumed one, so u == total maps to the EOF block
    __device__ __forceinline__ uint64_t voff(uint64_t u) const
    {
        const uint64_t total = rec_off[n];
        if (u >= total) return (header_bytes + blk_off[(total + BAI_BLOCK - 1u) / BAI_BLOCK]) << 16;
        return ((header_bytes + blk_off[u / BAI_BLOCK]) << 16) | (u % BAI_BLOCK);
    }
    // the file size as a virtual offset: what the reader reports after the EOF block
    __device__ __forceinline__ uint64_t final_off() const
    {
        return (header_bytes + blk_off[(rec_off[n] + BAI_BLOCK - 1u) / BAI_BLOCK] + 28u) << 16;
    }
    // start of record i, or the file's end for i == n
    __device__ __forceinline__ uint64_t start(uint32_t i) const { return i < n ? voff(rec_off[i]) : final_off(); }
};

struct BaiRec {
    uint32_t* ref;                // refID (BAI_NO_REF: unplaced, or refID >= n_refs)
    uint32_t* pos;
    uint32_t* bin;
    uint64_t* pm;                 // refID:end of a mapped record, refID:0 otherwise; scanned to the prefix maximum
    uint32_t* mapped;             // [n + 1] 1 for a mapped placed record; scanned to counts
    uint32_t* status;             // [2] bit c set: status code c applies; the number of unplaced records
};

__global__ void __launch_bounds__(128)
bai_record_kernel(const uint8_t* __restrict__ recs, const BaiFile f, const uint32_t n_refs, const BaiRec r)
{
    const uint32_t i = blockIdx.x * 128u + threadIdx.x;
    bool unplaced = false;
    if (i < f.n) {
        const uint64_t s = f.rec_off[i], len = f.rec_off[i + 1u] - s;
        const uint8_t* p = recs + s;
        const uint64_t key = sort_key(p, len);
        uint32_t bad = 0u;
        if (i > 0u) {
            const uint64_t s0 = f.rec_off[i - 1u];
            if (sort_key(recs + s0, s - s0) > key) bad |= 1u << 1;
        }
        const uint32_t ref = (uint32_t)(key >> 32), pos = (uint32_t)key;
        unplaced = ref == BAI_NO_REF;
        uint32_t rlen = 0u, flag = 0x4u;
        if (len >= BAM_FIXED) {
            const uint32_t l_name = p[12], n_cigar = (uint32_t)p[16] | ((uint32_t)p[17] << 8);
            flag = (uint32_t)p[18] | ((uint32_t)p[19] << 8);
            for (uint32_t k = 0; k < n_cigar && BAM_FIXED + l_name + 4u * (uint64_t)(k + 1u) <= len; ++k) {
                const uint32_t c = get32(p + BAM_FIXED + l_name + 4u * k), op = c & 15u;
                if (op == 0u || op == 2u || op == 3u || op == 7u || op == 8u) rlen += c >> 4;     // M D N = X
            }
        }
        if (rlen == 0u) rlen = 1u;
        uint32_t bin = BAI_UNPLACED_BIN, out_ref = BAI_NO_REF;
        uint64_t end = 0u;
        if (!unplaced) {
            if (ref >= n_refs) bad |= 1u << 2;
            end = (uint64_t)pos + rlen;
            if ((int32_t)pos < 0 || end > (1ull << 29)) { bad |= 1u << 3; end = (uint64_t)1u << 29; }
            else bin = bam_reg2bin(pos, (int64_t)end);
            if (ref < n_refs) out_ref = ref;
        }
        const bool mapped = out_ref != BAI_NO_REF && !(flag & 0x4u);
        r.ref[i] = out_ref; r.pos[i] = pos; r.bin[i] = bin;
        r.pm[i] = ((uint64_t)out_ref << 32) | (mapped ? end : 0u);
        r.mapped[i] = mapped;
        if (bad) atomicOr(r.status, bad);
    }
    if (i == 0u) r.mapped[f.n] = 0u;
    const uint32_t u = __popc(__ballot_sync(0xFFFFFFFFu, unplaced));
    if ((threadIdx.x & 31u) == 0u && u) atomicAdd(r.status + 1, u);
}

// run heads of equal (refID, bin) over placed records, and each refID's record range [first, last)
__global__ void __launch_bounds__(128)
bai_head_kernel(const uint32_t* __restrict__ ref, const uint32_t* __restrict__ bin, const uint32_t n, uint32_t* __restrict__ head,
                uint32_t* __restrict__ first, uint32_t* __restrict__ last)
{
    const uint32_t i = blockIdx.x * 128u + threadIdx.x;
    if (i > n) return;
    if (i == n) { head[n] = 0u; return; }
    const uint32_t r = ref[i];
    const bool new_ref = i == 0u || ref[i - 1u] != r;
    head[i] = r != BAI_NO_REF && (new_ref || bin[i - 1u] != bin[i]);
    if (r == BAI_NO_REF) return;
    if (new_ref) first[r] = i;
    if (i + 1u == n || ref[i + 1u] != r) last[r] = i + 1u;
}

struct BaiChunks {
    uint32_t* rec;                // first record of chunk c
    uint64_t* beg;
    uint64_t* end;
    uint32_t* owner;              // the bin that holds chunk c
    uint32_t* ref;
};

__global__ void __launch_bounds__(128)
bai_chunk_kernel(const BaiFile f, const uint32_t* __restrict__ head, const uint32_t* __restrict__ cidx, const uint32_t* __restrict__ ref,
                 const uint32_t* __restrict__ bin, const BaiChunks c)
{
    const uint32_t i = blockIdx.x * 128u + threadIdx.x;
    if (i < f.n && head[i]) { const uint32_t k = cidx[i]; c.rec[k] = i; c.owner[k] = bin[i]; c.ref[k] = ref[i]; }
}

// chunk k: [start of its first record, start of the next chunk's first record when that is on the same refID, else of the record after
// the refID's last one (or the file's end)); the sort keys refID:bin
__global__ void __launch_bounds__(128)
bai_chunk_fill_kernel(const BaiFile f, const uint32_t* __restrict__ cidx, const uint32_t* __restrict__ last, const BaiChunks c,
                      uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint32_t k = blockIdx.x * 128u + threadIdx.x, C = cidx[f.n];
    if (k >= f.n) return;
    vals[k] = k;
    if (k >= C) { keys[k] = ~0ull; return; }
    const uint32_t r = c.ref[k];
    const uint32_t next = k + 1u < C && c.ref[k + 1u] == r ? c.rec[k + 1u] : max(last[r], c.rec[k] + 1u);
    c.beg[k] = f.start(c.rec[k]);
    c.end[k] = f.start(min(next, f.n));
    keys[k] = ((uint64_t)r << 16) | c.owner[k];
}

__global__ void __launch_bounds__(128)
bai_rekey_kernel(const uint32_t n, const uint32_t* __restrict__ count, const BaiChunks c, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint32_t k = blockIdx.x * 128u + threadIdx.x;
    if (k >= n) return;
    vals[k] = k;
    keys[k] = k < *count ? ((uint64_t)c.ref[k] << 16) | c.owner[k] : ~0ull;
}

__device__ __forceinline__ uint32_t lower_bound64(const uint64_t* a, uint32_t lo, uint32_t hi, uint64_t x)
{
    while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2u; if (a[m] < x) lo = m + 1u; else hi = m; }
    return lo;
}

// compress_binning's pass over level l (bins [first, next_first)): a bin whose chunks (sorted by start) span fewer than 65536 compressed
// bytes moves them to its parent when the parent holds chunks of its own
__global__ void __launch_bounds__(128)
bai_level_kernel(const uint32_t* __restrict__ count, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                 const uint64_t* __restrict__ orig, const uint32_t lo_bin, const uint32_t hi_bin, const BaiChunks c, const uint32_t n)
{
    const uint32_t j = blockIdx.x * 128u + threadIdx.x, C = *count;
    if (j >= min(C, n)) return;
    const uint64_t key = keys[j];
    const uint32_t b = (uint32_t)(key & 0xFFFFu);
    if (b < lo_bin || b >= hi_bin) return;
    const uint32_t h = lower_bound64(keys, 0u, C, key), e = lower_bound64(keys, h, C, key + 1u);
    if ((c.end[vals[e - 1u]] >> 16) - (c.beg[vals[h]] >> 16) >= 65536u) return;
    const uint64_t pk = (key & ~0xFFFFull) | ((b - 1u) >> 3);
    const uint32_t p = lower_bound64(orig, 0u, C, pk);
    if (p < C && orig[p] == pk) c.owner[vals[j]] = (b - 1u) >> 3;
}

// a chunk that starts in the BGZF block where the previous chunk of its bin ends joins it (the chunks of a refID are disjoint and in file
// order, so the joined end is the later one's)
__global__ void __launch_bounds__(128)
bai_absorb_kernel(const uint32_t* __restrict__ count, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const BaiChunks c,
                  const uint32_t n, uint32_t* __restrict__ keep)
{
    const uint32_t j = blockIdx.x * 128u + threadIdx.x, C = min(*count, n);
    if (j > n) return;
    keep[j] = j < C && (j == 0u || keys[j - 1u] != keys[j] || (c.end[vals[j - 1u]] >> 16) < (c.beg[vals[j]] >> 16));
}

struct BaiOut {
    uint64_t* key;                // refID:bin of output chunk k, sorted
    uint64_t* beg;
    uint64_t* end;
    uint32_t* bin_head;           // [n + 1] 1 at the first chunk of a bin, 0 past the last chunk; scanned to the bins before chunk k
};

__global__ void __launch_bounds__(128)
bai_compact_kernel(const uint32_t* __restrict__ count, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                   const uint32_t* __restrict__ keep, const uint32_t* __restrict__ kpos, const BaiChunks c, const uint32_t n, const BaiOut o,
                   uint32_t* __restrict__ kb, uint32_t* __restrict__ ke)
{
    const uint32_t j = blockIdx.x * 128u + threadIdx.x, C = min(*count, n);
    if (j >= C) return;
    const uint32_t k = kpos[j] + keep[j] - 1u;                           // the output chunk that chunk j joins
    const uint32_t r = (uint32_t)(keys[j] >> 16);
    if (keep[j]) {
        o.key[k] = keys[j]; o.beg[k] = c.beg[vals[j]];
        o.bin_head[k] = j == 0u || keys[j - 1u] != keys[j];
        if (j == 0u || (uint32_t)(keys[j - 1u] >> 16) != r) kb[r] = k;
    }
    if (j + 1u == C || keep[j + 1u]) {
        o.end[k] = c.end[vals[j]];
        if (j + 1u == C || (uint32_t)(keys[j + 1u] >> 16) != r) ke[r] = k + 1u;
    }
}

struct BaiRefs {
    const uint32_t* first;        // record range [first, last) of refID r; first == last: no record
    const uint32_t* last;
    const uint32_t* kb;           // output chunk range [kb, ke)
    const uint32_t* ke;
    uint64_t* size;               // [n_refs + 1] bytes of refID r's part
    uint64_t* off;                // [n_refs + 1] its exclusive scan: where that part starts after the 8-byte head
};

__device__ __forceinline__ uint32_t n_intv(const BaiRec& r, const uint32_t first, const uint32_t last)
{
    if (first >= last) return 0u;
    const uint32_t end = (uint32_t)r.pm[last - 1u];
    return end ? ((end - 1u) >> 14) + 1u : 0u;
}

__global__ void __launch_bounds__(128)
bai_ref_size_kernel(const uint32_t n_refs, const BaiRec rec, const BaiRefs R, const uint32_t* __restrict__ bins_before)
{
    const uint32_t r = blockIdx.x * 128u + threadIdx.x;
    if (r > n_refs) return;
    if (r == n_refs) { R.size[n_refs] = 0u; return; }
    const uint32_t f = R.first[r], l = R.last[r], kb = R.kb[r], ke = max(R.ke[r], kb);
    const bool present = f < l;
    R.size[r] = 4u + 8u * (uint64_t)(bins_before[ke] - bins_before[kb]) + 16u * (uint64_t)(ke - kb) + (present ? 40u : 0u) + 4u +
                8u * (uint64_t)n_intv(rec, f, l);
}

__device__ __forceinline__ uint32_t bai_status(const BaiRec& rec)
{
    const uint32_t bits = rec.status[0];
    return bits & 2u ? 1u : (bits & 4u ? 2u : (bits & 8u ? 3u : 0u));
}

__device__ __forceinline__ uint64_t bai_size(const uint32_t n_refs, const BaiRefs& R) { return 8u + R.off[n_refs] + 8u; }

// the status, the size, and when the index fits: its head (magic, n_ref) and tail (n_no_coor)
__global__ void __launch_bounds__(32)
bai_finish_kernel(const uint32_t n_refs, const BaiRec rec, const BaiRefs R, const nvb_bai_out o)
{
    const uint32_t st = bai_status(rec);
    const uint64_t size = bai_size(n_refs, R);
    if (threadIdx.x != 0u) return;
    *o.d_status = st;
    *o.d_size = st ? 0u : size;
    if (st || size > o.capacity) return;
    o.d_bai[0] = 'B'; o.d_bai[1] = 'A'; o.d_bai[2] = 'I'; o.d_bai[3] = 1u;
    put32(o.d_bai + 4, n_refs);
    put64(o.d_bai + size - 8u, rec.status[1]);
}

// output chunk k, and the bin's (bin, n_chunk) before its first chunk
__global__ void __launch_bounds__(128)
bai_chunk_write_kernel(const uint32_t n, const uint32_t n_refs, const uint32_t* __restrict__ kpos, const BaiRec rec, const BaiRefs R,
                       const BaiOut ko, const uint32_t* __restrict__ bins_before, const nvb_bai_out o)
{
    const uint32_t k = blockIdx.x * 128u + threadIdx.x, K = kpos[n];
    if (k >= K || bai_status(rec) || bai_size(n_refs, R) > o.capacity) return;
    const uint64_t key = ko.key[k];
    const uint32_t r = (uint32_t)(key >> 16), kb = R.kb[r];
    uint8_t* p = o.d_bai + 8u + R.off[r] + 4u + 8u * (uint64_t)(bins_before[k + 1u] - bins_before[kb]) + 16u * (uint64_t)(k - kb);
    put64(p, ko.beg[k]);
    put64(p + 8, ko.end[k]);
    if (ko.bin_head[k]) {
        put32(p - 8, (uint32_t)(key & 0xFFFFu));
        put32(p - 4, lower_bound64(ko.key, k, K, key + 1u) - k);
    }
}

// first record in [lo, hi) whose prefix maximum of mapped ends exceeds t
__device__ __forceinline__ uint32_t first_reaching(const uint64_t* pm, uint32_t lo, uint32_t hi, const uint32_t t)
{
    while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2u; if ((uint32_t)pm[m] <= t) lo = m + 1u; else hi = m; }
    return lo;
}

// BAI_REF_CTAS CTAs per refID (blockIdx.x): the first writes n_bin, the pseudo-bin and n_intv; all of them share the linear index.  Window
// w's entry is the start of the first mapped record covering it: the first record i whose prefix maximum of mapped ends passes w's start,
// if i begins in or before w.  Otherwise w is not covered and takes the entry of the last covered window before it, which is the last
// window the records before i reach, or the refID's first start.
__global__ void __launch_bounds__(128)
bai_ref_write_kernel(const BaiFile f, const uint32_t n_refs, const BaiRec rec, const BaiRefs R, const uint32_t* __restrict__ bins_before,
                     const uint32_t* __restrict__ mapped_before, const nvb_bai_out o)
{
    const uint32_t r = blockIdx.x, t = threadIdx.x + 128u * blockIdx.y;
    if (bai_status(rec) || bai_size(n_refs, R) > o.capacity) return;
    const uint32_t first = R.first[r], last = R.last[r], kb = R.kb[r], ke = max(R.ke[r], kb);
    const bool present = first < last;
    const uint32_t nb = bins_before[ke] - bins_before[kb];
    uint8_t* base = o.d_bai + 8u + R.off[r];
    uint8_t* lin = base + 4u + 8u * (uint64_t)nb + 16u * (uint64_t)(ke - kb);
    const uint64_t off_beg = present ? f.start(first) : 0u;
    if (t == 0u) {
        put32(base, nb + (present ? 1u : 0u));
        if (present) {
            const uint32_t m = mapped_before[last] - mapped_before[first];
            put32(lin, BAI_META_BIN); put32(lin + 4, 2u);
            put64(lin + 8, off_beg); put64(lin + 16, f.start(last));
            put64(lin + 24, m); put64(lin + 32, (uint64_t)(last - first) - m);
        }
    }
    if (present) lin += 40u;
    const uint32_t ni = n_intv(rec, first, last);
    if (t == 0u) put32(lin, ni);
    for (uint32_t w = t; w < ni; w += 128u * BAI_REF_CTAS) {
        const uint32_t i = first_reaching(rec.pm, first, last, w << 14);
        uint64_t v = off_beg;
        if (i < last && (rec.pos[i] >> 14) <= w) v = f.start(i);
        else if (i < last && i > first && (uint32_t)rec.pm[i - 1u] != 0u)
            v = f.start(first_reaching(rec.pm, first, last, (((uint32_t)rec.pm[i - 1u] - 1u) >> 14) << 14));
        put64(lin + 4u + 8u * (uint64_t)w, v);
    }
}

} // namespace nvb

using namespace nvb;

extern "C" int nvb_bam_sort(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n, const nvb_bam_sort_out* out, void* d_temp,
                            size_t* temp_bytes, void* stream)
{
    if (!out || !temp_bytes || !out->d_offsets || (out->capacity && !out->d_records) || ((uintptr_t)out->d_records & 15u)) return NVB_E_INVALID;
    if (n > 0x7FFFFFFEu || (n && (!d_records || !d_offsets))) return NVB_E_INVALID;
    const cudaStream_t s = as_stream(stream);
    if (n == 0u) {
        *temp_bytes = 0;
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_offsets, 0, sizeof(uint64_t), s));
        return NVB_OK;
    }
    size_t sort_bytes = 0, scan_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                                 (uint32_t*)nullptr, (int)n, 0, 64, s));
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n + 1, s));
    TempCarver tc(nullptr);
    tc.take<uint64_t>(n); tc.take<uint64_t>(n); tc.take<uint32_t>(n); tc.take<uint32_t>(n); tc.take<uint64_t>((size_t)n + 1);
    tc.take<char>(std::max(sort_bytes, scan_bytes));
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    TempCarver t(d_temp);
    uint64_t* keys = t.take<uint64_t>(n);
    uint64_t* keys_sorted = t.take<uint64_t>(n);
    uint32_t* idx = t.take<uint32_t>(n);
    uint32_t* order = out->d_order ? out->d_order : t.take<uint32_t>(n);
    if (out->d_order) t.take<uint32_t>(n);
    uint64_t* sizes = t.take<uint64_t>((size_t)n + 1);
    void* cub_tmp = t.take<char>(std::max(sort_bytes, scan_bytes));

    const uint32_t grid = (n + 127u) / 128u;
    bam_sort_key_kernel<<<grid, 128, 0, s>>>(d_records, d_offsets, n, keys, idx);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_bytes, keys, keys_sorted, idx, order, (int)n, 0, 64, s));
    bam_sort_size_kernel<<<(n + 1u + 127u) / 128u, 128, 0, s>>>(d_offsets, order, n, sizes);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, scan_bytes, sizes, out->d_offsets, (int)n + 1, s));
    if (out->capacity == 0u) return NVB_OK;
    bam_gather_kernel<<<(n + SORT_RUN - 1u) / SORT_RUN, SORT_THREADS, 0, s>>>(d_records, d_offsets, order, out->d_offsets, n, out->d_records,
                                                                               out->capacity);
    return (int)cudaGetLastError();
}

extern "C" int nvb_bam_index(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n, const uint64_t* d_block_offsets,
                             uint64_t header_bytes, uint32_t n_refs, uint32_t max_ref_len, const nvb_bai_out* out, void* d_temp,
                             size_t* temp_bytes, void* stream)
{
    if (!out || !temp_bytes || !out->d_size || !out->d_status || (out->capacity && !out->d_bai)) return NVB_E_INVALID;
    if (!d_offsets || !d_block_offsets || (n && !d_records) || n > 0x7FFFFFFEu || n_refs > 0x7FFFFFFEu) return NVB_E_INVALID;
    if (max_ref_len > (1u << 29)) return NVB_E_UNSUPPORTED;
    const cudaStream_t s = as_stream(stream);
    const size_t nr = std::max<size_t>(n, 1u), nrefs = std::max<uint32_t>(n_refs, 1u);
    uint32_t bw = 1u;
    while (bw < 32u && (n_refs >> bw)) ++bw;
    const int end_bit = 16 + (int)bw;                                    // refID:bin keys; the padding key ~0 sorts last

    size_t sort_bytes = 0, scan32 = 0, scan64 = 0, max_bytes = 0, cub_bytes;
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                                 (uint32_t*)nullptr, (int)nr, 0, end_bit, s));
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan32, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)nr + 1, s));
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan64, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)nrefs + 1, s));
    NVB_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, max_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, cub::Max(), (int)nr, s));
    cub_bytes = std::max(std::max(sort_bytes, scan32), std::max(scan64, max_bytes));

    auto carve = [&](TempCarver& t, BaiRec& rec, BaiChunks& ch, BaiOut& ko, uint64_t*& kA, uint64_t*& kB, uint64_t*& orig, uint32_t*& vA,
                     uint32_t*& vB, uint32_t*& head, uint32_t*& cidx, uint32_t*& keep, uint32_t*& kpos, uint32_t*& bins_before,
                     uint32_t*& mapped_before, uint32_t*& first, uint32_t*& last, uint32_t*& kb, uint32_t*& ke, uint64_t*& rsize,
                     uint64_t*& roff, void*& cub_tmp) {
        rec.ref = t.take<uint32_t>(nr); rec.pos = t.take<uint32_t>(nr); rec.bin = t.take<uint32_t>(nr); rec.pm = t.take<uint64_t>(nr);
        rec.mapped = t.take<uint32_t>(nr + 1); rec.status = t.take<uint32_t>(2);
        mapped_before = t.take<uint32_t>(nr + 1); head = t.take<uint32_t>(nr + 1); cidx = t.take<uint32_t>(nr + 1);
        ch.rec = t.take<uint32_t>(nr); ch.beg = t.take<uint64_t>(nr); ch.end = t.take<uint64_t>(nr); ch.owner = t.take<uint32_t>(nr);
        ch.ref = t.take<uint32_t>(nr);
        kA = t.take<uint64_t>(nr); kB = t.take<uint64_t>(nr); orig = t.take<uint64_t>(nr); vA = t.take<uint32_t>(nr); vB = t.take<uint32_t>(nr);
        keep = t.take<uint32_t>(nr + 1); kpos = t.take<uint32_t>(nr + 1);
        ko.key = t.take<uint64_t>(nr); ko.beg = t.take<uint64_t>(nr); ko.end = t.take<uint64_t>(nr); ko.bin_head = t.take<uint32_t>(nr + 1);
        bins_before = t.take<uint32_t>(nr + 1);
        first = t.take<uint32_t>(nrefs); last = t.take<uint32_t>(nrefs); kb = t.take<uint32_t>(nrefs); ke = t.take<uint32_t>(nrefs);
        rsize = t.take<uint64_t>(nrefs + 1); roff = t.take<uint64_t>(nrefs + 1);
        cub_tmp = t.take<char>(cub_bytes);
    };
    BaiRec rec; BaiChunks ch; BaiOut ko;
    uint64_t *kA, *kB, *orig, *rsize, *roff;
    uint32_t *vA, *vB, *head, *cidx, *keep, *kpos, *bins_before, *mapped_before, *first, *last, *kb, *ke;
    void* cub_tmp;
    {
        TempCarver tc(nullptr);
        carve(tc, rec, ch, ko, kA, kB, orig, vA, vB, head, cidx, keep, kpos, bins_before, mapped_before, first, last, kb, ke, rsize, roff, cub_tmp);
        const size_t need = tc.total();
        if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    }
    TempCarver t(d_temp);
    carve(t, rec, ch, ko, kA, kB, orig, vA, vB, head, cidx, keep, kpos, bins_before, mapped_before, first, last, kb, ke, rsize, roff, cub_tmp);

    BaiFile f;
    f.rec_off = d_offsets; f.blk_off = d_block_offsets; f.header_bytes = header_bytes; f.n = n;
    BaiRefs R;
    R.first = first; R.last = last; R.kb = kb; R.ke = ke; R.size = rsize; R.off = roff;
    const uint32_t gn = (uint32_t)((nr + 1u + 127u) / 128u);             // n + 1 threads
    NVB_CUDA_TRY(cudaMemsetAsync(rec.status, 0, 2 * sizeof(uint32_t), s));
    NVB_CUDA_TRY(cudaMemsetAsync(first, 0, 4 * nrefs, s));
    NVB_CUDA_TRY(cudaMemsetAsync(last, 0, 4 * nrefs, s));
    NVB_CUDA_TRY(cudaMemsetAsync(kb, 0, 4 * nrefs, s));
    NVB_CUDA_TRY(cudaMemsetAsync(ke, 0, 4 * nrefs, s));
    NVB_CUDA_TRY(cudaMemsetAsync(ko.bin_head, 0, 4 * (nr + 1), s));
    if (n == 0u) {
        NVB_CUDA_TRY(cudaMemsetAsync(cidx, 0, 4 * (nr + 1), s));
        NVB_CUDA_TRY(cudaMemsetAsync(kpos, 0, 4 * (nr + 1), s));
        NVB_CUDA_TRY(cudaMemsetAsync(bins_before, 0, 4 * (nr + 1), s));
        NVB_CUDA_TRY(cudaMemsetAsync(mapped_before, 0, 4 * (nr + 1), s));
    } else {
        bai_record_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(d_records, f, n_refs, rec);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::InclusiveScan(cub_tmp, cub_bytes, rec.pm, rec.pm, cub::Max(), (int)n, s));
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, rec.mapped, mapped_before, (int)n + 1, s));
        bai_head_kernel<<<gn, 128, 0, s>>>(rec.ref, rec.bin, n, head, first, last);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, head, cidx, (int)n + 1, s));
        bai_chunk_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(f, head, cidx, rec.ref, rec.bin, ch);
        NVB_LAUNCH_CHECK();
        bai_chunk_fill_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(f, cidx, last, ch, kA, vA);
        NVB_LAUNCH_CHECK();
        const uint32_t* C = cidx + n;
        NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, kA, orig, vA, vB, (int)n, 0, end_bit, s));
        const uint64_t* cur = orig;
        for (uint32_t l = 5u; l >= 1u; --l) {                            // compress_binning's level passes, finest first
            const uint32_t lo_bin = ((1u << (3u * l)) - 1u) / 7u, hi_bin = ((1u << (3u * l + 3u)) - 1u) / 7u;
            bai_level_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(C, cur, vB, orig, lo_bin, hi_bin, ch, n);
            NVB_LAUNCH_CHECK();
            bai_rekey_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(n, C, ch, kA, vA);
            NVB_LAUNCH_CHECK();
            NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, kA, kB, vA, vB, (int)n, 0, end_bit, s));
            cur = kB;
        }
        bai_absorb_kernel<<<gn, 128, 0, s>>>(C, kB, vB, ch, n, keep);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, keep, kpos, (int)n + 1, s));
        bai_compact_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(C, kB, vB, keep, kpos, ch, n, ko, kb, ke);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, ko.bin_head, bins_before, (int)n + 1, s));
    }
    if (n_refs) {
        bai_ref_size_kernel<<<(n_refs + 1u + 127u) / 128u, 128, 0, s>>>(n_refs, rec, R, bins_before);
        NVB_LAUNCH_CHECK();
        NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, rsize, roff, (int)n_refs + 1, s));
    } else {
        NVB_CUDA_TRY(cudaMemsetAsync(roff, 0, sizeof(uint64_t), s));
    }
    bai_finish_kernel<<<1, 32, 0, s>>>(n_refs, rec, R, *out);
    NVB_LAUNCH_CHECK();
    if (out->capacity == 0u) return NVB_OK;
    if (n) {
        bai_chunk_write_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(n, n_refs, kpos, rec, R, ko, bins_before, *out);
        NVB_LAUNCH_CHECK();
    }
    if (n_refs) {
        bai_ref_write_kernel<<<dim3(n_refs, BAI_REF_CTAS), 128, 0, s>>>(f, n_refs, rec, R, bins_before, mapped_before, *out);
        NVB_LAUNCH_CHECK();
    }
    return NVB_OK;
}
