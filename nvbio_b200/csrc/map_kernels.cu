// map_kernels.cu -- nvBowtie's seed mapping stage as a batch primitive (SURVEY 8a row a10 / 8f-2):
//
//   nvb_map_seeds          map_queues_kernel<EXACT_MAPPING | APPROX_MAPPING>   nvBowtie/bowtie2/cuda/mapping_inl.h:229-316, 318-366, 539-591
//                          + the bounded per-read priority deque of SeedHits    seed_hit.h:54-98,230-244, seed_hit_deque_array.h:157-204,
//                                                                               mapping_inl.h:99-115 (store_deque)
//   nvb_fm_locate_init /   the two-phase locate of queued SA rows               locate_inl.h:122-210 (locate_init_kernel / locate_lookup_kernel),
//   nvb_fm_locate_lookup /                                                      nvbio/fmindex/fmindex_inl.h:502-569 (locate_ssa_iterator / lookup_ssa_iterator)
//   nvb_fm_locate_sorted   the same with the rows radix-sorted first            aligner_best_approx.h:737-756 (sort the SA rows to gather locality)
//
// Design.  One thread per queued read (as the reference), but the hits go straight into the read's slot of the output arena, kept
// SORTED by range size (ascending, stable in push order) -- the order pop_top() returns them in -- instead of a 512-entry
// local-memory interval heap copied out afterwards.  The reference's bounded push ("deque full -> pop_bottom(), then push") is
// reproduced literally: when the slot holds max_hits entries its LAST one (a largest range; the most recently pushed among equal
// sizes) is dropped and the new hit inserted at its sorted place.  Which of several equally large ranges an interval heap would
// have dropped is a property of that heap's internal layout; the multiset of range sizes kept, the push counts and the
// range_sum / range_count statistics are identical, and so are the complete hit sets whenever a read produces at most max_hits
// hits (the common case: 100 slots for ~30-60 seeds).
#include "fm_core.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace nvb {

struct MapGeom {
    uint32_t algorithm, seed_len, seed_freq, max_hits, retry_stride, rep_seeds, subseed_len, min_read_len, fw, rc, retry;
};

__device__ __forceinline__ uint32_t hit_bits(uint32_t delta, uint32_t pos, uint32_t rc, uint32_t indexdir)
{
    return (delta & 0xFFFFFu) | ((pos & 0x3FFu) << 20) | ((rc & 1u) << 30) | ((indexdir & 1u) << 31);   // SeedHit bit-fields, seed_hit.h:230-232
}

// bounded, sorted push (see the header comment); range is INCLUSIVE here and stored exclusive like SeedHit (utils.h:52-53)
struct HitSlot {
    nvb_seed_hit* data; uint32_t n, cap;
    __device__ __forceinline__ void push(uint32_t x, uint32_t y, uint32_t pos, uint32_t rc)
    {
        if (cap == 0u) return;
        if (n == cap) --n;                                            // pop_bottom(): drop a largest range
        const uint32_t delta = y + 1u - x;                            // exclusive range [x, y+1): delta = size
        uint32_t i = n;
        while (i > 0u && (data[i - 1u].bits & 0xFFFFFu) > (delta & 0xFFFFFu)) { data[i] = data[i - 1u]; --i; }
        nvb_seed_hit h; h.range_begin = x; h.bits = hit_bits(delta, pos, rc, 0u);
        data[i] = h;
        ++n;
    }
};

template <int BITS>
__global__ void __launch_bounds__(128)
map_seeds_kernel(const FmIndex f, const StrSet reads, const uint32_t* __restrict__ queue, const uint32_t n_queue, const MapGeom g,
                 const uint32_t* __restrict__ seed_freq_per_read,
                 nvb_seed_hit* __restrict__ hits, uint32_t* __restrict__ counts, uint8_t* __restrict__ reseed, uint32_t* __restrict__ stats)
{
    const uint32_t id = blockIdx.x * 128 + threadIdx.x;
    if (id >= n_queue) return;
    const uint32_t read_id = queue ? queue[id] : id;
    const uint32_t begin = str_off(reads, read_id), read_len = str_len(reads, read_id);
    if (read_len < g.min_read_len) { counts[read_id] = 0u; return; }           // (the reference leaves reseed[id] untouched here too)

    const uint32_t seed_len  = g.seed_len < read_len ? g.seed_len : read_len;
    const uint32_t seed_freq = seed_freq_per_read ? seed_freq_per_read[read_id] : g.seed_freq;
    const uint32_t stride    = seed_freq_per_read ? seed_freq / (g.retry_stride ? g.retry_stride : 1u) : (g.retry_stride ? g.seed_freq / g.retry_stride : 0u);
    HitSlot slot; slot.data = hits + (size_t)read_id * g.max_hits; slot.n = 0u; slot.cap = g.max_hits;
    uint32_t range_sum = 0u, range_count = 0u;
    SymReader<BITS, true> rd(reads.words);

    // seed positions relative to the read: begin + read_len is 2^32 for a read ending on the stream's last symbol
    for (uint32_t rel = g.retry * stride; rel + seed_len <= read_len; rel += (seed_freq ? seed_freq : 1u)) {
        const uint32_t pos = begin + rel;
        // seeds with N's: BOTH mappers skip a seed with any N.  The approximate one asks util::count_occurrences(seed, len, 4, 2) -- which
        // returns the COUNT (capped at 2), not "count >= 2" -- inside an if(): one N already makes it true (mapping_inl.h:258, 343-346;
        // nvbio/basic/numbers.h:108-122), so map()'s own single-N handling is never reached from here
        uint32_t n_cnt = 0u;
        for (uint32_t i = 0; i < seed_len; ++i) n_cnt += (rd.get(pos + i) > 3u) ? 1u : 0u;
        if (n_cnt >= 1u) continue;
        const uint32_t pos_fw = read_len - rel - seed_len, pos_rc = rel;        // SeedHit::m_pos of the two strands (:267, :301)
        if (g.algorithm == NVB_MAP_EXACT) {
            uint32_t x, y;
            if (g.fw) {
                fm_match_one<BITS, true>(f, reads.words, pos, seed_len, NVB_MATCH_FORWARD_ORDER, x, y);
                if (x <= y) { slot.push(x, y, pos_fw, 0u); range_sum += y - x + 1u; ++range_count; }
            }
            if (g.rc) {
                fm_match_one<BITS, true>(f, reads.words, pos, seed_len, NVB_MATCH_COMPLEMENT, x, y);
                if (x <= y) { slot.push(x, y, pos_rc, 1u); range_sum += y - x + 1u; ++range_count; }
            }
        } else {
            // map<CHECK_EXACT>(forward reader) then map<IGNORE_EXACT>(reversed + complemented reader), subseed exact (:347-364)
            uint2 tmp[NVB_MAP_MAX_PUSHES];
            for (uint32_t strand = 0; strand < 2u; ++strand) {
                if (strand == 0u ? !g.fw : !g.rc) continue;
                uint32_t sum = 0u;
                const uint32_t n = fm_map_approx_one<BITS, true>(f, reads.words, pos, seed_len, g.subseed_len,
                                                                strand == 0u ? NVB_MATCH_FORWARD_ORDER : NVB_MATCH_COMPLEMENT, strand == 0u,
                                                                tmp, NVB_MAP_MAX_PUSHES, sum);
                const uint32_t m = n < NVB_MAP_MAX_PUSHES ? n : NVB_MAP_MAX_PUSHES;
                for (uint32_t k = 0; k < m; ++k) slot.push(tmp[k].x, tmp[k].y, strand == 0u ? pos_fw : pos_rc, strand);
                range_sum += sum; range_count += n;
            }
        }
    }
    counts[read_id] = slot.n;
    if (reseed) reseed[id] = (range_count == 0u || range_sum >= g.rep_seeds * range_count) ? 1 : 0;      // mapping_inl.h:586-588
    if (stats) { stats[2u * id] = range_sum; stats[2u * id + 1u] = range_count; }
}

// ---- two-phase locate ---------------------------------------------------------------------------------------------------------
// locate_ssa_iterator: walk LF until a sampled row; returns (that row, steps)            fmindex_inl.h:502-538
__device__ __forceinline__ uint2 fm_locate_init_one(const FmIndex& f, uint32_t row)
{
    uint32_t j = row, t = 0;
    while ((j & f.sa_mask) != 0u) {
        if (j != f.primary) {
            const uint32_t k = j < f.primary ? j : j - 1u;
            const FmBlock b = load_block(f.blocks, k >> 6);
            const uint32_t c = block_symbol(b, k & 63u);
            j = f.l2(c) + block_rank(b, k & 63u, c);
        } else j = 0u;
        ++t;
    }
    return make_uint2(j, t);
}

__global__ void __launch_bounds__(256)
locate_init_kernel(const FmIndex f, const uint32_t* __restrict__ rows, const uint32_t* __restrict__ idx, uint32_t n,
                   uint32_t* __restrict__ out_row, uint32_t* __restrict__ out_steps)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = idx ? idx[t] : t;
    const uint2 r = fm_locate_init_one(f, rows[i]);
    out_row[i] = r.x; out_steps[i] = r.y;
}
__global__ void __launch_bounds__(256)
locate_lookup_kernel(const FmIndex f, const uint32_t* __restrict__ rows, const uint32_t* __restrict__ steps, const uint32_t* __restrict__ idx,
                     uint32_t n, uint32_t* __restrict__ pos)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = idx ? idx[t] : t;
    pos[i] = gather_u32(f.ssa + (rows[i] >> f.sa_shift)) + steps[i];             // lookup_ssa_iterator, fmindex_inl.h:553-569
}
__global__ void __launch_bounds__(256)
iota_kernel(uint32_t* __restrict__ v, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t < n) v[t] = t;
}
// rows arrive sorted; position of sorted entry t goes back to its original slot idx[t]
__global__ void __launch_bounds__(256)
locate_sorted_kernel(const FmIndex f, const uint32_t* __restrict__ sorted_rows, const uint32_t* __restrict__ idx, uint32_t n, uint32_t* __restrict__ pos)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    pos[idx[t]] = fm_locate_one(f, sorted_rows[t]);
}

} // namespace nvb

using namespace nvb;

extern "C" int nvb_map_seeds(const nvb_fm_index* fmi, const nvb_string_set* reads, const uint32_t* d_queue, uint32_t n_queue, uint32_t retry,
                             const nvb_map_params* P, const uint32_t* d_seed_freq,
                             nvb_seed_hit* d_hits, uint32_t* d_counts, uint8_t* d_reseed, uint32_t* d_range_stats, void* stream)
{
    if (!valid_fmindex(fmi) || !valid_strset(reads) || !P || (n_queue && (!d_hits || !d_counts))) return NVB_E_INVALID;
    if (reads->bits == 8 || !reads->big_endian) return NVB_E_UNSUPPORTED;
    if (P->algorithm != NVB_MAP_EXACT && P->algorithm != NVB_MAP_APPROX) return NVB_E_UNSUPPORTED;      // case pruning needs the reverse index
    if (P->seed_len == 0 || P->max_hits == 0 || P->max_hits > 0xFFFFFu || (!d_seed_freq && P->seed_freq == 0)) return NVB_E_INVALID;
    if (P->algorithm == NVB_MAP_APPROX && 3u * P->seed_len + 1u > NVB_MAP_MAX_PUSHES) return NVB_E_UNSUPPORTED;
    if (n_queue == 0) return NVB_OK;
    nvb_fm_index plain = *fmi;
    if (P->algorithm == NVB_MAP_APPROX) { plain.d_ktab = nullptr; plain.ktab_k = 0; }
    const FmIndex f = make_fmindex(&plain);
    MapGeom g;
    g.algorithm = P->algorithm; g.seed_len = P->seed_len; g.seed_freq = P->seed_freq; g.max_hits = P->max_hits;
    g.retry_stride = P->max_reseed + 1u; g.rep_seeds = P->rep_seeds; g.subseed_len = P->subseed_len; g.min_read_len = P->min_read_len;
    g.fw = P->fw; g.rc = P->rc; g.retry = retry;
    const StrSet rs = make_strset(reads);
    const uint32_t grid = (n_queue + 127u) / 128u;
    if (rs.bits == 2) map_seeds_kernel<2><<<grid, 128, 0, as_stream(stream)>>>(f, rs, d_queue, n_queue, g, d_seed_freq, d_hits, d_counts, d_reseed, d_range_stats);
    else              map_seeds_kernel<4><<<grid, 128, 0, as_stream(stream)>>>(f, rs, d_queue, n_queue, g, d_seed_freq, d_hits, d_counts, d_reseed, d_range_stats);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

extern "C" int nvb_fm_locate_init(const nvb_fm_index* fmi, const uint32_t* d_rows, const uint32_t* d_idx, uint32_t n,
                                  uint32_t* d_sampled_row, uint32_t* d_steps, void* stream)
{
    if (!valid_fmindex(fmi) || (n && (!d_rows || !d_sampled_row || !d_steps))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    locate_init_kernel<<<(n + 255u) / 256u, 256, 0, as_stream(stream)>>>(make_fmindex(fmi), d_rows, d_idx, n, d_sampled_row, d_steps);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

extern "C" int nvb_fm_locate_lookup(const nvb_fm_index* fmi, const uint32_t* d_sampled_row, const uint32_t* d_steps, const uint32_t* d_idx, uint32_t n,
                                    uint32_t* d_pos, void* stream)
{
    if (!valid_fmindex(fmi) || !fmi->d_ssa || (n && (!d_sampled_row || !d_steps || !d_pos))) return NVB_E_INVALID;
    if (n == 0) return NVB_OK;
    locate_lookup_kernel<<<(n + 255u) / 256u, 256, 0, as_stream(stream)>>>(make_fmindex(fmi), d_sampled_row, d_steps, d_idx, n, d_pos);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}

extern "C" int nvb_fm_locate_sorted(const nvb_fm_index* fmi, const uint32_t* d_rows, uint32_t n, uint32_t* d_pos,
                                    void* d_temp, size_t* temp_bytes, void* stream)
{
    if (!valid_fmindex(fmi) || !fmi->d_ssa || !temp_bytes || (n && (!d_rows || !d_pos))) return NVB_E_INVALID;
    TempCarver tc(d_temp);
    uint32_t* keys_out = tc.take<uint32_t>(n);
    uint32_t* idx_in   = tc.take<uint32_t>(n);
    uint32_t* idx_out  = tc.take<uint32_t>(n);
    size_t sort_bytes = 0;
    int end_bit = 32; { uint32_t v = fmi->length; end_bit = 1; while ((v >>= 1) != 0u) ++end_bit; }
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_rows, keys_out, idx_in, idx_out, (int)n, 0, end_bit, as_stream(stream)));
    char* sort_tmp = tc.take<char>(sort_bytes);
    const size_t need = tc.total();
    if (!d_temp || *temp_bytes < need) { *temp_bytes = need; return NVB_E_TEMP_SIZE; }
    if (n == 0) return NVB_OK;
    cudaStream_t s = as_stream(stream);
    const uint32_t grid = (n + 255u) / 256u;
    iota_kernel<<<grid, 256, 0, s>>>(idx_in, n);
    NVB_LAUNCH_CHECK();
    NVB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, d_rows, keys_out, idx_in, idx_out, (int)n, 0, end_bit, s));
    locate_sorted_kernel<<<grid, 256, 0, s>>>(make_fmindex(fmi), keys_out, idx_out, n, d_pos);
    NVB_LAUNCH_CHECK();
    return NVB_OK;
}
