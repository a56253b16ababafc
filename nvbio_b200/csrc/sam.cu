// sam.cu -- nvb_sam_format: SAM text of BAM records in device memory.  Three steps, as bam.cu:
//   sam_size_kernel   one thread per record: its validity and exact line length (sam_line_size, sam_core.cuh) into sizes, with the
//                     extra 0 element, and the rejection tally (warp-reduced, one atomic per warp);
//   an exclusive scan of the sizes into d_offsets (CUB);
//   sam_write_kernel  a CTA takes SAM_RUN consecutive records.  Both their input records and their output lines are contiguous, so the
//                     CTA loads the run's records into a shared span with aligned 16-byte loads, its warps compose the lines (a warp per
//                     record, sam_compose) into a second shared span laid out like the output modulo 16, and the CTA stores that span
//                     with aligned 16-byte stores (bytes only at the partial lines at either end).  A record whose input or line is
//                     larger than its span is composed directly from and to global memory.
#include <cub/cub.cuh>
#include "sam_core.cuh"

namespace nvb {

constexpr uint32_t SAM_RUN = 32u;                   // records per CTA of the write kernel
constexpr uint32_t SAM_IN_STAGE = 16384u;           // bytes of its input span
constexpr uint32_t SAM_OUT_STAGE = 24576u;          // bytes of its output span

__global__ void __launch_bounds__(128)
sam_size_kernel(const uint8_t* __restrict__ records, const uint64_t* __restrict__ in_off, const uint32_t n, const uint32_t n_refs,
                const uint32_t* __restrict__ ref_off, uint64_t* __restrict__ sizes, uint32_t* __restrict__ rejected)
{
    const uint32_t i = blockIdx.x * 128u + threadIdx.x;
    bool bad = false;
    if (i < n) {
        const uint64_t b = in_off[i], e = in_off[i + 1];
        const uint64_t s = e >= b ? sam_line_size(records + b, e - b, n_refs, ref_off) : 0u;
        sizes[i] = s;
        bad = s == 0u;
    }
    if (i == 0u) sizes[n] = 0u;                     // the scan's extra element: d_offsets[n] = the total
    const uint32_t nbad = __reduce_add_sync(0xFFFFFFFFu, bad ? 1u : 0u);
    const uint32_t first = __reduce_min_sync(0xFFFFFFFFu, bad ? i : 0xFFFFFFFFu);
    if ((threadIdx.x & 31u) == 0u && nbad) {
        atomicAdd(rejected, nbad);
        atomicMin(rejected + 1, first);
    }
}

// copy global bytes [lo, hi) (addresses of `g`, shifted so that g + x is 16-byte aligned when x is) to s + (x - base): whole 16-byte
// lines as uint4, the partial lines at either end byte by byte.  `s` + base - lo keeps the output's alignment modulo 16.
__device__ __forceinline__ void sam_copy_span(uint8_t* __restrict__ dst, uint64_t dbase, const uint8_t* __restrict__ src, uint64_t sbase,
                                              uint64_t lo, uint64_t hi, bool to_global)
{
    const uint64_t a0 = (lo + 15u) & ~(uint64_t)15u, a1 = hi & ~(uint64_t)15u;
    if (a0 >= a1) {
        for (uint64_t g = lo + threadIdx.x; g < hi; g += 128u) dst[g - dbase] = src[g - sbase];
        return;
    }
    for (uint64_t g = lo + threadIdx.x; g < a0; g += 128u) dst[g - dbase] = src[g - sbase];
    for (uint64_t g = a0 + 16u * threadIdx.x; g < a1; g += 16u * 128u) {
        if (to_global) *(uint4*)(dst + (g - dbase)) = *(const uint4*)(src + (g - sbase));
        else           *(uint4*)(dst + (g - dbase)) = __ldg((const uint4*)(src + (g - sbase)));
    }
    for (uint64_t g = a1 + threadIdx.x; g < hi; g += 128u) dst[g - dbase] = src[g - sbase];
}

// records0 / text0: d_records / d_text rounded down to 16 bytes, with imis / omis the bytes they were rounded by, so that input byte x
// is records0[x + imis] and output byte y is text0[y + omis]
__global__ void __launch_bounds__(128)
sam_write_kernel(const uint8_t* __restrict__ records0, const uint32_t imis, const uint64_t* __restrict__ in_off, const uint32_t n,
                 const char* __restrict__ ref_names, const uint32_t* __restrict__ ref_off, const uint64_t* __restrict__ out_off,
                 uint8_t* __restrict__ text0, const uint32_t omis, const uint64_t capacity)
{
    __shared__ __align__(16) uint8_t istage[SAM_IN_STAGE];
    __shared__ __align__(16) uint8_t ostage[SAM_OUT_STAGE];
    __shared__ uint64_t si[SAM_RUN + 1u], so[SAM_RUN + 1u];
    const uint32_t r0 = blockIdx.x * SAM_RUN, r1 = min(n, r0 + SAM_RUN);
    if (r0 >= r1) return;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = threadIdx.x; i <= r1 - r0; i += 128u) { si[i] = in_off[r0 + i] + imis; so[i] = out_off[r0 + i] + omis; }
    __syncthreads();
    const uint64_t cap = capacity + omis;
    // lines that fit the capacity are a prefix: line k is stored when out_off[k + 1] <= capacity
    for (uint32_t r = r0; r < r1 && so[r + 1u - r0] <= cap;) {
        const uint64_t ib = si[r - r0] & ~(uint64_t)15u, ob = so[r - r0] & ~(uint64_t)15u;
        uint32_t e = r + 1u;
        while (e < r1 && so[e + 1u - r0] <= cap && si[e + 1u - r0] >= si[e - r0] && si[e + 1u - r0] - ib <= SAM_IN_STAGE &&
               so[e + 1u - r0] - ob <= SAM_OUT_STAGE)
            ++e;
        if (si[e - r0] < si[r - r0] || si[e - r0] - ib > SAM_IN_STAGE || so[e - r0] - ob > SAM_OUT_STAGE) {
            // record r alone is larger than a span (or, rejected, has no extent): composed from and to global memory
            const uint64_t size = so[r + 1u - r0] - so[r - r0];
            if (warp == 0u && size)
                sam_compose(records0 + si[r - r0], size, ref_names, ref_off, (char*)text0 + so[r - r0], lane, 32u);
            r = e;
            continue;
        }
        sam_copy_span(istage, ib, records0, 0u, si[r - r0], si[e - r0], false);
        __syncthreads();
        for (uint32_t k = r + warp; k < e; k += 4u) {
            const uint64_t size = so[k + 1u - r0] - so[k - r0];
            if (size) sam_compose(istage + (si[k - r0] - ib), size, ref_names, ref_off, (char*)ostage + (so[k - r0] - ob), lane, 32u);
        }
        __syncthreads();
        sam_copy_span(text0, 0u, ostage, ob, so[r - r0], so[e - r0], true);
        __syncthreads();
        r = e;
    }
}

} // namespace nvb

using namespace nvb;

extern "C" int nvb_sam_format(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n,
                              const char* d_ref_names, const uint32_t* d_ref_name_offsets, uint32_t n_refs,
                              const nvb_sam_out* out, void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!out || !temp_bytes || !out->d_offsets || !out->d_rejected || (out->capacity && !out->d_text)) return NVB_E_INVALID;
    if ((n && (!d_records || !d_offsets)) || (n_refs && (!d_ref_names || !d_ref_name_offsets)) || n >= 0x7FFFFFFFu) return NVB_E_INVALID;
    const cudaStream_t s = as_stream(stream);
    if (n == 0u) {
        *temp_bytes = 0;
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_offsets, 0, sizeof(uint64_t), s));
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_rejected, 0, sizeof(uint32_t), s));
        NVB_CUDA_TRY(cudaMemsetAsync(out->d_rejected + 1, 0xFF, sizeof(uint32_t), s));
        return NVB_OK;
    }
    size_t scan_bytes = 0;
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n + 1, s));
    TempCarver tc(nullptr);
    tc.take<uint64_t>((size_t)n + 1); tc.take<char>(scan_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    TempCarver t(d_temp);
    uint64_t* sizes = t.take<uint64_t>((size_t)n + 1);
    void* scan_tmp = t.take<char>(scan_bytes);

    NVB_CUDA_TRY(cudaMemsetAsync(out->d_rejected, 0, sizeof(uint32_t), s));
    NVB_CUDA_TRY(cudaMemsetAsync(out->d_rejected + 1, 0xFF, sizeof(uint32_t), s));
    sam_size_kernel<<<(n + 127u) / 128u, 128, 0, s>>>(d_records, d_offsets, n, n_refs, d_ref_name_offsets, sizes, out->d_rejected);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, sizes, out->d_offsets, (int)n + 1, s));
    if (out->capacity == 0u) return NVB_OK;
    const uint32_t imis = (uint32_t)((uintptr_t)d_records & 15u), omis = (uint32_t)((uintptr_t)out->d_text & 15u);
    sam_write_kernel<<<(n + SAM_RUN - 1u) / SAM_RUN, 128, 0, s>>>(d_records - imis, imis, d_offsets, n, d_ref_names, d_ref_name_offsets,
                                                                  out->d_offsets, (uint8_t*)out->d_text - omis, omis, out->capacity);
    return (int)cudaGetLastError();
}
