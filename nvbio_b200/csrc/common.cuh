// common.cuh -- shared device/host helpers for the nvbio_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include "../../include/nvbio_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "nvbio_b200 kernels are written for sm_90a (H100) only"
#endif

namespace nvb {

constexpr int NVB_MAX_DEVICES = 64;      // per-device state (function attributes, stage events) is kept in arrays of this size

#define NVB_CUDA_TRY(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) return (int)_e; } while (0)
#define NVB_LAUNCH_CHECK() do { cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return (int)_e; } while (0)

static inline cudaStream_t as_stream(void* s) { return (cudaStream_t)s; }

// SMs of the current device (132 on an H100 SXM), cached per device: resident grids that stride over a device-side count are
// sized from it.  1 if the device cannot be queried (the launch that follows reports the error; a grid is never empty).
static inline uint32_t sm_count() {
    static std::atomic<uint32_t> cached[NVB_MAX_DEVICES];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= NVB_MAX_DEVICES) return 1u;
    uint32_t n = cached[dev].load(std::memory_order_relaxed);
    if (n == 0u) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 1u;
        n = (uint32_t)v;
        cached[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// carve sub-buffers out of a caller-provided temp allocation
struct TempCarver {
    char*  base; size_t off;
    explicit TempCarver(void* p) : base((char*)p), off(0) {}
    template <typename T> T* take(size_t count) {
        off = align_up(off, 256);
        T* r = base ? (T*)(base + off) : (T*)nullptr;
        off += count * sizeof(T);
        return r;
    }
    size_t total() const { return align_up(off, 256); }
};

// ---------------------------------------------------------------------------------------------
// packed symbol streams (PackedStream semantics, nvbio/basic/packedstream_inl.h:336-372)
// ---------------------------------------------------------------------------------------------
struct StrSet {
    const uint32_t* words;
    const uint32_t* offsets;
    const uint32_t* lengths;
    uint32_t bits, big_endian, stride, length;
};

static inline StrSet make_strset(const nvb_string_set* s) {
    StrSet r;
    r.words = s->d_words; r.offsets = s->d_offsets; r.lengths = s->d_lengths;
    r.bits = s->bits; r.big_endian = s->big_endian; r.stride = s->stride; r.length = s->length;
    return r;
}
static inline bool valid_strset(const nvb_string_set* s) {
    return s && s->d_words && (s->bits == 2 || s->bits == 4 || s->bits == 8);
}
// a known pairing policy and no unknown flag bit (nvb_pair_params)
static inline bool valid_pair_policy(const nvb_pair_params* pp) {
    return pp->policy <= NVB_PE_RR && (pp->flags & ~(NVB_PE_NO_OVERLAP | NVB_PE_DISCORDANT | NVB_PE_NO_MIXED)) == 0u;
}

__host__ __device__ __forceinline__ uint32_t str_off(const StrSet& s, uint32_t i) { return s.offsets ? s.offsets[i] : i * s.stride; }
__host__ __device__ __forceinline__ uint32_t str_len(const StrSet& s, uint32_t i) { return s.lengths ? s.lengths[i] : s.length; }

// symbol p of a packed stream.  BITS in {2,4,8}.  8-bit streams are plain byte arrays.
template <int BITS, bool BE>
__host__ __device__ __forceinline__ uint32_t sym_from_word(uint32_t w, uint32_t p) {
    constexpr uint32_t SPW = 32 / BITS;
    const uint32_t r = p & (SPW - 1);
    const uint32_t sh = BE ? (32 - BITS - BITS * r) : (BITS * r);
    return (w >> sh) & ((1u << BITS) - 1u);
}
template <int BITS, bool BE>
__host__ __device__ __forceinline__ uint32_t sym_at(const uint32_t* __restrict__ words, uint32_t p) {
    if (BITS == 8) return ((const uint8_t*)words)[p];
    constexpr uint32_t LOG_SPW = (BITS == 2) ? 4 : 3;
    return sym_from_word<BITS, BE>(words[p >> LOG_SPW], p);
}
__host__ __device__ __forceinline__ uint32_t sym_at_rt(const uint32_t* __restrict__ words, uint32_t bits, uint32_t be, uint32_t p) {
    if (bits == 8) return ((const uint8_t*)words)[p];
    if (bits == 2) return be ? sym_at<2, true>(words, p) : sym_at<2, false>(words, p);
    return be ? sym_at<4, true>(words, p) : sym_at<4, false>(words, p);
}

// A tiny sequential reader that keeps the current word in a register (one global load per
// 16 / 8 / 4 symbols when walking monotonically in either direction).
template <int BITS, bool BE>
struct SymReader {
    const uint32_t* words;
    uint32_t cur_idx, cur_word;
    __host__ __device__ __forceinline__ explicit SymReader(const uint32_t* w) : words(w), cur_idx(0xFFFFFFFFu), cur_word(0) {}
    __host__ __device__ __forceinline__ uint32_t get(uint32_t p) {
        constexpr uint32_t LOG_SPW = (BITS == 2) ? 4 : (BITS == 4 ? 3 : 2);
        const uint32_t wi = p >> LOG_SPW;
        if (wi != cur_idx) { cur_idx = wi; cur_word = words[wi]; }
        if (BITS == 8) return (cur_word >> (8 * (p & 3))) & 0xFFu;   // byte order = memory order
        return sym_from_word<BITS, BE>(cur_word, p);
    }
};

// nvb_bgzf_compress with the byte count in device memory (bgzf.cu): d_n_bytes (NULL = n_bytes) holds the count, n_bytes is a host upper
// bound that sizes the grids, the temp and d_block_offsets ([ceil(n_bytes / 0xFF00) + 1] entries; those past the real members repeat the
// total).  nvb_bgzf_compress is this call with d_n_bytes = NULL.  Only its first kernel reads d_in, and only its last one writes d_out, so
// d_out may overlap d_in (never the temp): the BAM pipeline writes the members over the records they compress
int bgzf_compress_device_count(const uint8_t* d_in, uint64_t n_bytes, const uint64_t* d_n_bytes, const nvb_bgzf_out* out, void* d_temp,
                               size_t* temp_bytes, void* stream);

// dispatch a callable templated on <BITS,BE> from runtime (bits, big_endian)
#define NVB_DISPATCH_STREAM(bits, be, CALL)                         \
    do {                                                            \
        if ((bits) == 2) { if (be) { CALL(2, true); } else { CALL(2, false); } } \
        else if ((bits) == 4) { if (be) { CALL(4, true); } else { CALL(4, false); } } \
        else { CALL(8, false); }                                    \
    } while (0)

} // namespace nvb
