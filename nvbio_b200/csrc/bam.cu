// bam.cu -- nvb_bam_records: BAM alignment records of traced and finished alignments in device memory.  Three steps:
//   bam_plan_kernel     one thread per read (per pair when paired, so both mates' placement is decided in one place): the record cores
//                       and sizes (bam_plan_unit, bam_core.cuh) and the tallies;
//   an exclusive scan   of the sizes into d_offsets (CUB);
//   bam_write_kernel    a CTA takes BAM_RUN consecutive records, which are contiguous in the output; its warps compose them (a warp per
//                       record, bam_compose) into a shared-memory span laid out like the output modulo 16, which the CTA then stores with
//                       aligned 16-byte stores (bytes only at the head and tail).  Records start at arbitrary byte offsets, so a thread
//                       writing its own record byte by byte would touch 32 lines per warp store.  A record larger than the span is
//                       composed directly in the output.
#include <cub/cub.cuh>
#include "bam_core.cuh"

namespace nvb {

constexpr uint32_t BAM_RUN = 64u;                   // records per CTA of the write kernel
constexpr uint32_t BAM_STAGE = 32768u;              // bytes of its staging span

__global__ void __launch_bounds__(128)
bam_plan_kernel(const BamIn in, const uint32_t n_units, uint32_t* __restrict__ cores, uint64_t* __restrict__ sizes, uint32_t* __restrict__ counts)
{
    const uint32_t u = blockIdx.x * 128u + threadIdx.x;
    uint32_t cnt[3] = { 0u, 0u, 0u }, recs = 0u;
    if (u < n_units) {
        bam_plan_unit(in, u, cores, sizes, cnt);
        recs = in.pair_flags ? 2u : 1u;
    }
    if (u == 0u) sizes[in.n] = 0u;                  // the scan's extra element: d_offsets[n] = the total
    recs = __reduce_add_sync(0xFFFFFFFFu, recs);
    cnt[0] = __reduce_add_sync(0xFFFFFFFFu, cnt[0]);
    cnt[1] = __reduce_add_sync(0xFFFFFFFFu, cnt[1]);
    cnt[2] = __reduce_add_sync(0xFFFFFFFFu, cnt[2]);
    if ((threadIdx.x & 31u) == 0u && recs) {
        atomicAdd(counts, recs);
        if (cnt[0]) atomicAdd(counts + 1, cnt[0]);
        if (cnt[1]) atomicAdd(counts + 2, cnt[1]);
        if (cnt[2]) atomicAdd(counts + 3, cnt[2]);
    }
}

template <int BITS, bool BE>
__global__ void __launch_bounds__(128)
bam_write_kernel(const BamIn in, const uint32_t* __restrict__ cores, const uint64_t* __restrict__ offsets, uint8_t* __restrict__ out, const uint64_t capacity,
                 const uint32_t* __restrict__ d_n)
{
    __shared__ __align__(16) uint8_t stage[BAM_STAGE];
    __shared__ uint64_t so[BAM_RUN + 1u];
    const uint32_t n = d_n ? min(*d_n, in.n) : in.n;         // nvb_bam_records_all: the record count lives on the device
    const uint32_t r0 = blockIdx.x * BAM_RUN, r1 = min(n, r0 + BAM_RUN);
    if (r0 >= r1) return;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = threadIdx.x; i <= r1 - r0; i += 128u) so[i] = offsets[r0 + i];
    __syncthreads();
    // records that fit the capacity are a prefix: record k is stored when offsets[k + 1] <= capacity
    for (uint32_t r = r0; r < r1 && so[r + 1u - r0] <= capacity;) {
        const uint64_t base = so[r - r0] & ~(uint64_t)15u;
        uint32_t e = r + 1u;
        while (e < r1 && so[e + 1u - r0] <= capacity && so[e + 1u - r0] - base <= BAM_STAGE) ++e;
        if (so[e - r0] - base > BAM_STAGE) {         // record r alone is larger than the span
            if (warp == 0u)
                bam_compose<BITS, BE>(in, r, cores + 8u * (size_t)r, (uint32_t)(so[r + 1u - r0] - so[r - r0]), out + so[r - r0], lane, 32u);
            r = e;
            continue;
        }
        for (uint32_t k = r + warp; k < e; k += 4u)
            bam_compose<BITS, BE>(in, k, cores + 8u * (size_t)k, (uint32_t)(so[k + 1u - r0] - so[k - r0]), stage + (so[k - r0] - base), lane, 32u);
        __syncthreads();
        // store [lo, hi): whole 16-byte lines from the span, the partial lines at either end byte by byte
        const uint64_t lo = so[r - r0], hi = so[e - r0];
        const uint64_t a0 = (lo + 15u) & ~(uint64_t)15u, a1 = hi & ~(uint64_t)15u;
        if (a0 >= a1) {
            for (uint64_t g = lo + threadIdx.x; g < hi; g += 128u) out[g] = stage[g - base];
        } else {
            for (uint64_t g = lo + threadIdx.x; g < a0; g += 128u) out[g] = stage[g - base];
            for (uint64_t g = a0 + 16u * threadIdx.x; g < a1; g += 16u * 128u)
                *(uint4*)(out + g) = *(const uint4*)(stage + (g - base));
            for (uint64_t g = a1 + threadIdx.x; g < hi; g += 128u) out[g] = stage[g - base];
        }
        __syncthreads();
        r = e;
    }
}

// nvb_bam_records_all, one thread per read: pass 1 (rec_first == NULL) its record count and the tallies, pass 2 its records' plans
__global__ void __launch_bounds__(128)
bam_all_plan_kernel(const BamIn in, const uint32_t n_reads, const uint32_t* __restrict__ first, const uint32_t capacity,
                    const uint32_t* __restrict__ rec_first, uint4* rec, uint32_t* __restrict__ n_rec, uint32_t* __restrict__ cores,
                    uint64_t* __restrict__ sizes, uint32_t* __restrict__ counts)
{
    const uint32_t r = blockIdx.x * 128u + threadIdx.x;
    uint32_t cnt[3] = { 0u, 0u, 0u };
    if (r < n_reads) {
        const uint32_t m = bam_plan_read_all(in, r, first, capacity, rec_first, rec, cores, sizes, cnt);
        if (!rec_first) n_rec[r] = m;
        else if (r == n_reads - 1u) counts[0] = rec_first[n_reads];
    }
    if (rec_first) return;
    cnt[0] = __reduce_add_sync(0xFFFFFFFFu, cnt[0]);
    cnt[1] = __reduce_add_sync(0xFFFFFFFFu, cnt[1]);
    cnt[2] = __reduce_add_sync(0xFFFFFFFFu, cnt[2]);
    if ((threadIdx.x & 31u) == 0u) {
        if (cnt[0]) atomicAdd(counts + 1, cnt[0]);
        if (cnt[1]) atomicAdd(counts + 2, cnt[1]);
        if (cnt[2]) atomicAdd(counts + 3, cnt[2]);
    }
}

} // namespace nvb

using namespace nvb;

// the BamIn of an nvb_bam_in (n = alignments, or record slots)
static BamIn make_bam_in(const nvb_bam_in* in, uint32_t n)
{
    const nvb_finish_out& F = in->finish;
    BamIn b;
    b.reads = make_strset(&in->reads); b.quals = in->d_read_quals;
    b.n_ops = in->d_n_ops; b.begin = (const uint2*)in->d_begin; b.strand = in->d_strand;
    b.cigar = F.d_cigar; b.max_cigar = F.max_cigar; b.n_cigar = F.d_n_cigar;
    b.md = F.d_md; b.max_md = F.max_md; b.md_len = F.d_md_len; b.edits = F.d_edits;
    b.score = in->d_score; b.mapq = in->d_mapq; b.second = in->d_second_score; b.pair_flags = in->d_pair_flags;
    b.contig_begin = in->d_contig_begin; b.n_contigs = in->n_contigs;
    b.names = in->d_names; b.name_off = in->d_name_offsets; b.n = n;
    return b;
}

// the argument checks both entry points share
static bool valid_bam_args(const nvb_bam_in* in, const nvb_bam_out* out, const size_t* temp_bytes)
{
    if (!in || !out || !temp_bytes) return false;
    const nvb_finish_out& F = in->finish;
    if (!valid_strset(&in->reads) || in->reads.bits == 8) return false;
    if (!in->d_n_ops || !in->d_begin || !in->d_strand || !F.d_cigar || !F.d_n_cigar || !F.d_md || !F.d_md_len || !F.d_edits ||
        F.max_cigar == 0u || F.max_md == 0u || !in->d_score || !in->d_contig_begin || in->n_contigs == 0u || !in->d_names || !in->d_name_offsets)
        return false;
    return out->d_offsets && out->d_counts && (!out->capacity || out->d_records) && !((uintptr_t)out->d_records & 15u);
}

template <typename L>
static void launch_write(const nvb_bam_in* in, L launch)
{
    if (in->reads.bits == 2) { if (in->reads.big_endian) launch(bam_write_kernel<2, true>); else launch(bam_write_kernel<2, false>); }
    else                     { if (in->reads.big_endian) launch(bam_write_kernel<4, true>); else launch(bam_write_kernel<4, false>); }
}

extern "C" int nvb_bam_records(const nvb_bam_in* in, uint32_t n, const nvb_bam_out* out, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!valid_bam_args(in, out, temp_bytes)) return NVB_E_INVALID;
    if ((in->d_pair_flags && (n & 1u)) || n > 0x7FFFFFFEu) return NVB_E_INVALID;
    const cudaStream_t s = as_stream(stream);
    if (n == 0u) {
        *temp_bytes = 0;
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_offsets, 0, sizeof(uint64_t), s));
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_counts, 0, 4 * sizeof(uint32_t), s));
        return NVB_OK;
    }
    size_t scan_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n + 1, s));
    TempCarver tc(nullptr);
    tc.take<uint32_t>(8 * (size_t)n); tc.take<uint64_t>((size_t)n + 1); tc.take<char>(scan_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    TempCarver t(d_temp);
    uint32_t* cores = t.take<uint32_t>(8 * (size_t)n);
    uint64_t* sizes = t.take<uint64_t>((size_t)n + 1);
    void* scan_tmp = t.take<char>(scan_bytes);

    const BamIn b = make_bam_in(in, n);

    const uint32_t units = in->d_pair_flags ? n / 2u : n;
    NVB_CUDA_TRY(cudaMemsetAsync(out->d_counts, 0, 4 * sizeof(uint32_t), s));
    bam_plan_kernel<<<(units + 127u) / 128u, 128, 0, s>>>(b, units, cores, sizes, out->d_counts);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, sizes, out->d_offsets, (int)n + 1, s));
    if (out->capacity == 0u) return NVB_OK;
    const uint32_t grid = (n + BAM_RUN - 1u) / BAM_RUN;
    launch_write(in, [&](auto kernel) { kernel<<<grid, 128, 0, s>>>(b, cores, out->d_offsets, out->d_records, out->capacity, nullptr); });
    return (int)cudaGetLastError();
}

extern "C" int nvb_bam_records_all(const nvb_bam_all_in* in, uint32_t n_reads, const nvb_bam_out* out, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!in || !valid_bam_args(&in->base, out, temp_bytes)) return NVB_E_INVALID;
    if (in->base.d_pair_flags || !in->d_first) return NVB_E_INVALID;
    const uint64_t slots64 = (uint64_t)n_reads + in->capacity;
    if (slots64 > 0x7FFFFFFEull) return NVB_E_INVALID;
    const uint32_t slots = (uint32_t)slots64;
    const cudaStream_t s = as_stream(stream);
    if (n_reads == 0u) {
        *temp_bytes = 0;
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_offsets, 0, sizeof(uint64_t), s));
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_counts, 0, 4 * sizeof(uint32_t), s));
        return NVB_OK;
    }
    size_t scan_bytes = 0, scan2 = 0;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)slots + 1, s));
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan2, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n_reads + 1, s));
    if (scan2 > scan_bytes) scan_bytes = scan2;
    TempCarver tc(nullptr);
    tc.take<uint32_t>(8 * (size_t)slots); tc.take<uint64_t>((size_t)slots + 1); tc.take<uint4>(slots); tc.take<uint32_t>((size_t)n_reads + 1);
    tc.take<uint32_t>((size_t)n_reads + 1); tc.take<char>(scan_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    TempCarver t(d_temp);
    uint32_t* cores = t.take<uint32_t>(8 * (size_t)slots);
    uint64_t* sizes = t.take<uint64_t>((size_t)slots + 1);
    uint4* rec = t.take<uint4>(slots);
    uint32_t* n_rec = t.take<uint32_t>((size_t)n_reads + 1);
    uint32_t* rec_first = t.take<uint32_t>((size_t)n_reads + 1);
    void* scan_tmp = t.take<char>(scan_bytes);

    // the per-alignment inputs (n_ops, begin, strand, score, finish outputs) are indexed by alignment, `reads`, names, MAPQ and second
    // score by read; records name their alignment and read in rec
    BamIn b = make_bam_in(&in->base, slots);
    b.rec = rec;
    const uint32_t grid = (n_reads + 127u) / 128u;
    NVB_CUDA_TRY(cudaMemsetAsync(out->d_counts, 0, 4 * sizeof(uint32_t), s));
    NVB_CUDA_TRY(cudaMemsetAsync(n_rec + n_reads, 0, sizeof(uint32_t), s));
    NVB_CUDA_TRY(cudaMemsetAsync(sizes, 0, sizeof(uint64_t) * ((size_t)slots + 1), s));      // slots past the records: size 0
    bam_all_plan_kernel<<<grid, 128, 0, s>>>(b, n_reads, in->d_first, in->capacity, nullptr, rec, n_rec, cores, sizes, out->d_counts);
    NVB_LAUNCH_CHECK();
    size_t sb = scan_bytes;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, sb, n_rec, rec_first, (int)n_reads + 1, s));
    bam_all_plan_kernel<<<grid, 128, 0, s>>>(b, n_reads, in->d_first, in->capacity, rec_first, rec, n_rec, cores, sizes, out->d_counts);
    NVB_LAUNCH_CHECK();
    sb = scan_bytes;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, sb, sizes, out->d_offsets, (int)slots + 1, s));
    if (out->capacity == 0u) return NVB_OK;
    const uint32_t wgrid = (slots + BAM_RUN - 1u) / BAM_RUN;
    launch_write(&in->base, [&](auto kernel) { kernel<<<wgrid, 128, 0, s>>>(b, cores, out->d_offsets, out->d_records, out->capacity, out->d_counts); });
    return (int)cudaGetLastError();
}
