// host_pipeline.cu -- nvb_pipeline: host buffers in, host buffers out, `depth` batches in flight.
//
// The reference hands batches from an input thread to one compute thread per device and synchronises the device after every
// stage (nvBowtie/bowtie2/cuda/compute_thread.cu:213-243, defs.h:64 optional_device_synchronize, aligner_best_approx.h:219-241).
// Here a batch is three stream-ordered steps -- H2D copy, nvb_seed_extend[_paired], D2H copy -- on a copy-in stream, the
// slot's own compute stream and a copy-out stream, chained by events; nothing blocks the host until wait().  Consecutive
// batches use different compute streams, so their kernels may share the SMs (the seed search leaves the integer pipes
// half idle, the extension leaves DRAM idle).
//
// BAM mode (nvb_pipeline_create_bam): the same slots, streams and events; a batch's compute step chains mapping with MAPQ and
// traceback -> finish -> BAM records [-> BGZF with the record total read on the device], all in one device allocation per slot whose
// stage buffers share bytes where their lifetimes do not overlap (bam_layout).  The counts leave on the copy-out stream with the batch;
// the payload, whose size only the device knows, is copied by wait (or by the submit that reuses an unwaited slot) with exactly its
// byte count, on a stream of its own so that it does not queue behind the copy-outs of later batches.
#include "common.cuh"
#include "../../include/nvbio_b200_debug.h"
#include <algorithm>
#include <cstdlib>
#include <new>
#include <vector>

using namespace nvb;

struct nvb_pipeline {
    int device;
    nvb_fm_index fmi; const uint32_t* d_genome; nvb_seed_extend_params params; nvb_pair_params pair; bool paired;
    uint32_t n_reads, read_len, wpr, bits, hit_capacity, depth;
    uint32_t n_compute;                 // compute streams shared round-robin by the slots (NVB_PIPELINE_COMPUTE_STREAMS, default 1)
    cudaStream_t compute[16];
    cudaStream_t h2d, d2h;
    struct Slot {
        cudaStream_t compute;
        uint32_t* d_in; void* d_temp; size_t temp_bytes;
        // device results (one allocation) and their pinned host mirror, same layout
        char *d_out, *h_out; size_t out_bytes;
        cudaEvent_t ev_in, ev_start, ev_done, ev_out;
        bool busy;
    };
    std::vector<Slot> slots;
    uint64_t next;
    // offsets into the out block
    size_t o_score, o_pos, o_nhits, o_pscore, o_pflags, o_mscore, o_mpos, o_mstrand, o_nrescue;

    // BAM mode: s.d_in is the slot's one allocation, s.d_out its fixed block (inside it), s.h_out the fixed block's pinned mirror
    bool bam;
    nvb_pipeline_bam_params bp; nvb_mapq_params mapq;
    uint32_t max_ops, max_cigar, max_md;
    cudaStream_t pay;                   // payload copies (synchronous for the host)
    struct BamSlot {
        uint32_t n;                     // reads of the batch in the slot
        bool filled, copied;            // a batch was submitted; its payload is in h_pay
        uint8_t* h_pay; size_t pay_cap;
        cudaEvent_t ev_pay;
    };
    std::vector<BamSlot> bslots;
    // offsets into a slot: inputs and per-read outputs, then the stage region at o_x
    size_t o_words, o_quals, o_lens, o_names, o_noff, o_fixed;
    size_t o_score1, o_pos1, o_second, o_mapq, o_nops, o_begin, o_strand;                       // single end
    size_t o_pair_score, o_pair_flags, o_second_pair, o_mate_second, o_mate_mapq;             // paired (+ o_score1 / o_pos1 / o_strand)
    size_t o_recoff, o_zoff;
    size_t o_x, x_ops, x_map, x_fin, x_cigar, x_ncigar, x_md, x_mdlen, x_edits, x_btemp, x_rec, x_ztemp, x_zout;
    size_t map_temp, bam_temp, z_temp, rec_cap, z_cap, slot_bytes;
    uint32_t z_blocks;                  // BGZF blocks of rec_cap bytes
};

// the fixed block of a BAM batch: what leaves the device with every batch
struct BamFixed {
    uint32_t n_hits[4];
    uint32_t n_rescue[2];
    uint32_t counts[4];
    uint32_t pad[2];
    uint64_t record_bytes;              // d_offsets[n] of nvb_bam_records
    uint64_t payload_z;                 // d_block_offsets[z_blocks] of the BGZF step: the compressed total
};

static void layout(nvb_pipeline* p, size_t* total)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { off = align_up(off, 256); const size_t o = off; off += bytes; return o; };
    const size_t n = p->n_reads;
    p->o_nhits = take(4 * sizeof(uint32_t));
    if (!p->paired) { p->o_score = take(n * sizeof(int32_t)); p->o_pos = take(n * sizeof(uint32_t)); }
    else {
        p->o_pscore = take(n / 2 * sizeof(int32_t)); p->o_pflags = take(n / 2 * sizeof(uint32_t));
        p->o_mscore = take(n * sizeof(int32_t)); p->o_mpos = take(n * sizeof(uint32_t)); p->o_mstrand = take(n);
        p->o_nrescue = take(2 * sizeof(uint32_t));
    }
    *total = align_up(off, 256);
}

static nvb_string_set reads_view(const nvb_pipeline* p, const uint32_t* d_words)
{
    nvb_string_set r;
    r.d_words = d_words; r.bits = p->bits; r.big_endian = 1; r.d_offsets = nullptr; r.d_lengths = nullptr;
    r.stride = p->wpr * (32u / p->bits); r.length = p->read_len;
    return r;
}

static int run_batch(nvb_pipeline* p, nvb_pipeline::Slot& s, size_t* temp_bytes, void* d_temp)
{
    const nvb_string_set rs = reads_view(p, s.d_in ? s.d_in : (const uint32_t*)16);
    char* o = s.d_out;
    if (!p->paired)
        return nvb_seed_extend(&p->fmi, p->d_genome, &rs, p->n_reads, &p->params, p->hit_capacity,
                               o ? (int32_t*)(o + p->o_score) : (int32_t*)16, o ? (uint32_t*)(o + p->o_pos) : (uint32_t*)16,
                               o ? (uint32_t*)(o + p->o_nhits) : nullptr, nullptr, nullptr, nullptr, nullptr, d_temp, temp_bytes, s.compute);
    nvb_pair_out po;
    po.d_pair_score = (int32_t*)(o + p->o_pscore); po.d_pair_flags = (uint32_t*)(o + p->o_pflags);
    po.d_mate_score = (int32_t*)(o + p->o_mscore); po.d_mate_pos = (uint32_t*)(o + p->o_mpos); po.d_mate_strand = (uint8_t*)(o + p->o_mstrand);
    po.d_n_rescue = (uint32_t*)(o + p->o_nrescue);
    return nvb_seed_extend_paired(&p->fmi, p->d_genome, &rs, p->n_reads / 2u, &p->params, p->hit_capacity, &p->pair, &po,
                                  (uint32_t*)(o + p->o_nhits), d_temp, temp_bytes, s.compute);
}

extern "C" void nvb_pipeline_destroy(nvb_pipeline* p)
{
    if (!p) return;
    int prev = 0; cudaGetDevice(&prev); cudaSetDevice(p->device);
    for (auto& b : p->bslots) {
        if (b.ev_pay) cudaEventSynchronize(b.ev_pay);
        if (b.h_pay) cudaFreeHost(b.h_pay);
        if (b.ev_pay) cudaEventDestroy(b.ev_pay);
    }
    if (p->pay) cudaStreamDestroy(p->pay);
    for (auto& s : p->slots) {
        if (s.compute) cudaStreamSynchronize(s.compute);
        if (s.d_in) cudaFree(s.d_in);
        if (s.d_temp) cudaFree(s.d_temp);
        if (s.d_out && !p->bam) cudaFree(s.d_out);                  // (BAM mode: inside d_in)
        if (s.h_out) cudaFreeHost(s.h_out);
        if (s.ev_in) cudaEventDestroy(s.ev_in);
        if (s.ev_start) cudaEventDestroy(s.ev_start);
        if (s.ev_done) cudaEventDestroy(s.ev_done);
        if (s.ev_out) cudaEventDestroy(s.ev_out);
    }
    for (uint32_t i = 0; i < p->n_compute; ++i) if (p->compute[i]) cudaStreamDestroy(p->compute[i]);
    if (p->h2d) cudaStreamDestroy(p->h2d);
    if (p->d2h) cudaStreamDestroy(p->d2h);
    cudaSetDevice(prev);
    delete p;
}

extern "C" int nvb_pipeline_create(const nvb_fm_index* fmi, const uint32_t* d_genome, const nvb_seed_extend_params* params,
                                   const nvb_pair_params* pair_params,
                                   uint32_t n_reads, uint32_t read_len, uint32_t words_per_read, uint32_t read_bits,
                                   uint32_t hit_capacity, uint32_t depth, nvb_pipeline** out)
{
    if (!fmi || !d_genome || !params || !out || n_reads == 0 || depth == 0 || depth > 16) return NVB_E_INVALID;
    if (!(read_bits == 2 || read_bits == 4) || (uint64_t)words_per_read * (32u / read_bits) < read_len) return NVB_E_INVALID;
    if (pair_params && (n_reads & 1u)) return NVB_E_INVALID;
    // every policy and flag but NVB_PE_DISCORDANT passes through to nvb_seed_extend_paired; the pipeline has no MAPQ stage to mark
    // discordant pairs with
    if (pair_params && (!valid_pair_policy(pair_params) || (pair_params->flags & NVB_PE_DISCORDANT))) return NVB_E_INVALID;
    nvb_pipeline* p = new (std::nothrow) nvb_pipeline();
    if (!p) return (int)cudaErrorMemoryAllocation;
    *out = nullptr;
    p->fmi = *fmi; p->d_genome = d_genome; p->params = *params; p->paired = pair_params != nullptr;
    if (pair_params) p->pair = *pair_params;
    p->n_reads = n_reads; p->read_len = read_len; p->wpr = words_per_read; p->bits = read_bits; p->hit_capacity = hit_capacity; p->depth = depth;
    p->h2d = p->d2h = nullptr; p->next = 0;
    p->n_compute = 1;
    if (const char* e = getenv("NVB_PIPELINE_COMPUTE_STREAMS")) { const int v = atoi(e); if (v >= 1) p->n_compute = (uint32_t)v; }
    if (p->n_compute > depth) p->n_compute = depth;
    for (int i = 0; i < 16; ++i) p->compute[i] = nullptr;
    int rc = NVB_OK;
#define PIPE_TRY(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { rc = (int)_e; goto fail; } } while (0)
    {
        PIPE_TRY(cudaGetDevice(&p->device));
        size_t out_bytes = 0; layout(p, &out_bytes);
        PIPE_TRY(cudaStreamCreateWithFlags(&p->h2d, cudaStreamNonBlocking));
        PIPE_TRY(cudaStreamCreateWithFlags(&p->d2h, cudaStreamNonBlocking));
        for (uint32_t i = 0; i < p->n_compute; ++i) PIPE_TRY(cudaStreamCreateWithFlags(&p->compute[i], cudaStreamNonBlocking));
        p->slots.resize(depth);
        for (auto& s : p->slots) { s = nvb_pipeline::Slot(); }
        uint32_t k = 0;
        for (auto& s : p->slots) {
            s.out_bytes = out_bytes; s.busy = false;
            s.compute = p->compute[k++ % p->n_compute];
            PIPE_TRY(cudaMalloc((void**)&s.d_in, (size_t)n_reads * words_per_read * sizeof(uint32_t) + 64));
            PIPE_TRY(cudaMalloc((void**)&s.d_out, out_bytes));
            PIPE_TRY(cudaHostAlloc((void**)&s.h_out, out_bytes, cudaHostAllocDefault));
            PIPE_TRY(cudaMemset(s.d_out, 0, out_bytes));
            PIPE_TRY(cudaEventCreateWithFlags(&s.ev_in, cudaEventDisableTiming));
            PIPE_TRY(cudaEventCreate(&s.ev_start));
            PIPE_TRY(cudaEventCreate(&s.ev_done));
            PIPE_TRY(cudaEventCreateWithFlags(&s.ev_out, cudaEventDisableTiming));
            size_t tb = 0;
            const int r = run_batch(p, s, &tb, nullptr);
            if (r != NVB_E_TEMP_SIZE) { rc = (r == NVB_OK) ? NVB_E_INVALID : r; goto fail; }
            s.temp_bytes = tb;
            PIPE_TRY(cudaMalloc(&s.d_temp, tb));
        }
    }
#undef PIPE_TRY
    *out = p;
    return NVB_OK;
fail:
    nvb_pipeline_destroy(p);
    return rc;
}

extern "C" int nvb_pipeline_submit(nvb_pipeline* p, const uint32_t* h_read_words, uint32_t* ticket)
{
    if (!p || !h_read_words || !ticket || p->bam) return NVB_E_INVALID;
    const uint32_t k = (uint32_t)(p->next % p->depth);
    nvb_pipeline::Slot& s = p->slots[k];
    if (s.busy) NVB_CUDA_TRY(cudaEventSynchronize(s.ev_out));        // the slot's previous results must have left the device
    // copy-in must not overwrite reads that the slot's previous kernels may still be reading
    NVB_CUDA_TRY(cudaStreamWaitEvent(p->h2d, s.ev_done, 0));
    NVB_CUDA_TRY(cudaMemcpyAsync(s.d_in, h_read_words, (size_t)p->n_reads * p->wpr * sizeof(uint32_t), cudaMemcpyHostToDevice, p->h2d));
    NVB_CUDA_TRY(cudaEventRecord(s.ev_in, p->h2d));
    NVB_CUDA_TRY(cudaStreamWaitEvent(s.compute, s.ev_in, 0));
    NVB_CUDA_TRY(cudaStreamWaitEvent(s.compute, s.ev_out, 0));       // ... nor may the kernels overwrite results still being copied out
    NVB_CUDA_TRY(cudaEventRecord(s.ev_start, s.compute));
    size_t tb = s.temp_bytes;
    const int r = run_batch(p, s, &tb, s.d_temp);
    if (r != NVB_OK) return r;
    NVB_CUDA_TRY(cudaEventRecord(s.ev_done, s.compute));
    NVB_CUDA_TRY(cudaStreamWaitEvent(p->d2h, s.ev_done, 0));
    NVB_CUDA_TRY(cudaMemcpyAsync(s.h_out, s.d_out, s.out_bytes, cudaMemcpyDeviceToHost, p->d2h));
    NVB_CUDA_TRY(cudaEventRecord(s.ev_out, p->d2h));
    s.busy = true;
    *ticket = k;
    ++p->next;
    return NVB_OK;
}

extern "C" int nvb_pipeline_wait(nvb_pipeline* p, uint32_t ticket, nvb_pipeline_result* out)
{
    if (!p || ticket >= p->depth || !out || p->bam) return NVB_E_INVALID;
    nvb_pipeline::Slot& s = p->slots[ticket];
    if (p->next == 0) return NVB_E_INVALID;                         // nothing was ever submitted
    if (s.busy) NVB_CUDA_TRY(cudaEventSynchronize(s.ev_out));       // (waiting twice for the same ticket returns the same buffers)
    s.busy = false;
    nvb_pipeline_result r = {};
    const char* h = s.h_out;
    r.n_hits = (const uint32_t*)(h + p->o_nhits);
    if (!p->paired) { r.best_score = (const int32_t*)(h + p->o_score); r.best_pos = (const uint32_t*)(h + p->o_pos); }
    else {
        r.pair_score = (const int32_t*)(h + p->o_pscore); r.pair_flags = (const uint32_t*)(h + p->o_pflags);
        r.mate_score = (const int32_t*)(h + p->o_mscore); r.mate_pos = (const uint32_t*)(h + p->o_mpos); r.mate_strand = (const uint8_t*)(h + p->o_mstrand);
        r.n_rescue = (const uint32_t*)(h + p->o_nrescue);
    }
    NVB_CUDA_TRY(cudaEventElapsedTime(&r.device_ms, s.ev_start, s.ev_done));
    *out = r;
    return NVB_OK;
}

extern "C" void nvb_pipeline_traffic(const nvb_pipeline* p, size_t* h2d_bytes, size_t* d2h_bytes)
{
    if (!p) return;
    if (p->bam) {
        const size_t n = p->n_reads, names = p->paired ? n / 2 : n;
        if (h2d_bytes) *h2d_bytes = n * p->wpr * sizeof(uint32_t) + (p->bp.has_quals ? n * p->wpr * (32u / p->bits) : 0) +
                                    (p->bp.has_lengths ? n * sizeof(uint32_t) : 0) + p->bp.max_name_bytes + (names + 1) * sizeof(uint32_t);
        if (d2h_bytes) *d2h_bytes = sizeof(BamFixed);
        return;
    }
    if (h2d_bytes) *h2d_bytes = (size_t)p->n_reads * p->wpr * sizeof(uint32_t);
    if (d2h_bytes) *d2h_bytes = p->slots.empty() ? 0 : p->slots[0].out_bytes;
}

// ---------------------------------------------------------------------------------------------
// BAM mode
// ---------------------------------------------------------------------------------------------

// the reads of a batch of n in a slot at `base`
static nvb_string_set bam_reads(const nvb_pipeline* p, const char* base)
{
    nvb_string_set r = reads_view(p, (const uint32_t*)(base + p->o_words));
    r.d_lengths = p->bp.has_lengths ? (const uint32_t*)(base + p->o_lens) : nullptr;
    return r;
}

static nvb_best_alignment_out bam_alignment(const nvb_pipeline* p, char* base)
{
    nvb_best_alignment_out a;
    a.d_ops = (uint8_t*)(base + p->o_x + p->x_ops); a.max_ops = p->max_ops;
    a.d_n_ops = (uint32_t*)(base + p->o_nops); a.d_begin = (nvb_uint2*)(base + p->o_begin); a.d_strand = (uint8_t*)(base + p->o_strand);
    return a;
}

// the mapping call of a batch of n reads (d_temp NULL: its size query)
static int bam_map(nvb_pipeline* p, char* base, uint32_t n, void* d_temp, size_t* temp_bytes, cudaStream_t st)
{
    const nvb_string_set rs = bam_reads(p, base);
    nvb_seed_extend_params ps = p->params;
    ps.d_read_quals = p->bp.has_quals ? (const uint8_t*)(base + p->o_quals) : nullptr;
    BamFixed* fx = (BamFixed*)(base + p->o_fixed);
    nvb_best_alignment_out ba = bam_alignment(p, base);
    if (!p->paired) {
        nvb_mapq_out mo;
        mo.d_second_score = (int32_t*)(base + p->o_second); mo.d_second_pos = nullptr; mo.d_second_strand = nullptr;
        mo.d_mapq = (uint8_t*)(base + p->o_mapq);
        return nvb_seed_extend_mapq(&p->fmi, p->d_genome, &rs, n, &ps, p->hit_capacity, (int32_t*)(base + p->o_score1),
                                    (uint32_t*)(base + p->o_pos1), fx->n_hits, nullptr, nullptr, nullptr, nullptr, &ba, &p->mapq, &mo,
                                    d_temp, temp_bytes, st);
    }
    ba.d_strand = nullptr;                                          // d_mate_strand holds it
    nvb_pair_out po;
    po.d_pair_score = (int32_t*)(base + p->o_pair_score); po.d_pair_flags = (uint32_t*)(base + p->o_pair_flags);
    po.d_mate_score = (int32_t*)(base + p->o_score1); po.d_mate_pos = (uint32_t*)(base + p->o_pos1);
    po.d_mate_strand = (uint8_t*)(base + p->o_strand); po.d_n_rescue = fx->n_rescue;
    nvb_pair_mapq_out mo;
    mo.d_second_pair_score = (int32_t*)(base + p->o_second_pair); mo.d_second_mate_pos = nullptr; mo.d_second_mate_strand = nullptr;
    mo.d_mate_second_score = (int32_t*)(base + p->o_mate_second); mo.d_mate_mapq = (uint8_t*)(base + p->o_mate_mapq);
    return nvb_seed_extend_paired_traceback(&p->fmi, p->d_genome, &rs, n / 2u, &ps, p->hit_capacity, &p->pair, &po, &ba, &p->mapq, &mo,
                                            fx->n_hits, d_temp, temp_bytes, st);
}

static nvb_finish_out bam_finish_out(const nvb_pipeline* p, char* base)
{
    char* x = base + p->o_x;
    nvb_finish_out f;
    f.d_cigar = (uint32_t*)(x + p->x_cigar); f.max_cigar = p->max_cigar; f.d_n_cigar = (uint32_t*)(x + p->x_ncigar);
    f.d_md = x + p->x_md; f.max_md = p->max_md; f.d_md_len = (uint32_t*)(x + p->x_mdlen); f.d_edits = (uint32_t*)(x + p->x_edits);
    return f;
}

// the records call of a batch of n reads (d_temp NULL: its size query)
static int bam_records(nvb_pipeline* p, char* base, uint32_t n, void* d_temp, size_t* temp_bytes, cudaStream_t st)
{
    nvb_bam_in in;
    in.reads = bam_reads(p, base);
    in.d_read_quals = p->bp.has_quals ? (const uint8_t*)(base + p->o_quals) : nullptr;
    in.d_n_ops = (const uint32_t*)(base + p->o_nops); in.d_begin = (const nvb_uint2*)(base + p->o_begin);
    in.d_strand = (const uint8_t*)(base + p->o_strand);
    in.finish = bam_finish_out(p, base);
    in.d_score = (const int32_t*)(base + p->o_score1);
    in.d_mapq = (const uint8_t*)(base + (p->paired ? p->o_mate_mapq : p->o_mapq));
    in.d_second_score = (const int32_t*)(base + (p->paired ? p->o_mate_second : p->o_second));
    in.d_pair_flags = p->paired ? (const uint32_t*)(base + p->o_pair_flags) : nullptr;
    in.d_contig_begin = p->bp.d_contig_begin; in.n_contigs = p->bp.n_contigs;
    in.d_names = base + p->o_names; in.d_name_offsets = (const uint32_t*)(base + p->o_noff);
    nvb_bam_out o;
    o.d_records = (uint8_t*)(base + p->o_x + p->x_rec); o.capacity = p->rec_cap;
    o.d_offsets = (uint64_t*)(base + p->o_recoff); o.d_counts = ((BamFixed*)(base + p->o_fixed))->counts;
    return nvb_bam_records(&in, n, &o, d_temp, temp_bytes, st);
}

// the BGZF step: the members of the d_offsets[n] record bytes (d_temp NULL: its size query)
static int bam_compress(nvb_pipeline* p, char* base, uint32_t n, void* d_temp, size_t* temp_bytes, cudaStream_t st)
{
    char* x = base + p->o_x;
    nvb_bgzf_out z;
    z.d_out = (uint8_t*)(x + p->x_zout); z.capacity = p->z_cap; z.d_block_offsets = (uint64_t*)(base + p->o_zoff);
    return bgzf_compress_device_count((const uint8_t*)(x + p->x_rec), p->rec_cap, (const uint64_t*)(base + p->o_recoff) + n, &z, d_temp,
                                      temp_bytes, st);
}

// Offsets of everything in a slot.  Inputs, the fixed block and the per-read outputs first; then the stage region, where
//   [0, O)                    traceback ops           live from the mapping call to finish
//   [O, O + T)                the mapping call's temp live during the mapping call
//   [max(O, R), + F)          finish outputs          live from finish to the records
//   after them, B             the records' temp       live during the records call
//   [0, R)                    records                 live from the records call to the end of BGZF's first kernel (or the payload
//                                                     copy without compress)
//   [0, Zo)                   BGZF members            written by BGZF's last kernel, after its first one has read the records
//   [max(R, Zo), + Zt)        BGZF temp               live during compression
// needs only the shapes: the three temp sizes are queried with addresses computed from a fake base
static int bam_layout(nvb_pipeline* p)
{
    const size_t n = p->n_reads, names = p->paired ? n / 2 : n, sym = (size_t)p->wpr * (32u / p->bits);
    size_t off = 0;
    auto take = [&](size_t bytes) { off = align_up(off, 256); const size_t o = off; off += bytes; return o; };
    p->o_words = take(n * p->wpr * sizeof(uint32_t));
    p->o_quals = take(p->bp.has_quals ? n * sym : 0);
    p->o_lens = take(p->bp.has_lengths ? n * sizeof(uint32_t) : 0);
    p->o_names = take(p->bp.max_name_bytes);
    p->o_noff = take((names + 1) * sizeof(uint32_t));
    p->o_fixed = take(sizeof(BamFixed));
    p->o_score1 = take(n * sizeof(int32_t)); p->o_pos1 = take(n * sizeof(uint32_t)); p->o_strand = take(n);
    p->o_nops = take(n * sizeof(uint32_t)); p->o_begin = take(n * sizeof(nvb_uint2));
    if (!p->paired) { p->o_second = take(n * sizeof(int32_t)); p->o_mapq = take(n); }
    else {
        p->o_pair_score = take(n / 2 * sizeof(int32_t)); p->o_pair_flags = take(n / 2 * sizeof(uint32_t));
        p->o_second_pair = take(n / 2 * sizeof(int32_t)); p->o_mate_second = take(n * sizeof(int32_t)); p->o_mate_mapq = take(n);
    }
    p->o_recoff = take((n + 1) * sizeof(uint64_t));
    // the record bound: every record at its largest (nvb_bam_records: 36 + l_name + 4 n_cigar + SEQ + QUAL + six integer tags of at
    // most 7 bytes + MD:Z of 4 + md_len bytes), the names' bytes once per record (twice per pair name when paired)
    const size_t L = p->read_len;
    p->rec_cap = align_up(n * (36 + 1 + 4 * (size_t)p->max_cigar + (L + 1) / 2 + L + 6 * 7 + 4 + p->max_md) +
                          (p->paired ? 2 : 1) * (size_t)p->bp.max_name_bytes, 256);
    p->z_blocks = (uint32_t)((p->rec_cap + 0xFEFFu) / 0xFF00u);
    p->z_cap = (size_t)65311 * p->z_blocks;
    p->o_zoff = take(p->bp.compress ? ((size_t)p->z_blocks + 1) * sizeof(uint64_t) : 0);
    p->o_x = align_up(off, 256);

    size_t x = 0;
    auto put = [&](size_t bytes) { x = align_up(x, 256); const size_t o = x; x += bytes; return o; };
    p->x_ops = 0;
    const size_t O = align_up(n * p->max_ops, 256);
    p->x_map = O;
    x = align_up(O > p->rec_cap ? O : p->rec_cap, 256);
    p->x_fin = x;
    p->x_cigar = put(n * p->max_cigar * sizeof(uint32_t)); p->x_ncigar = put(n * sizeof(uint32_t));
    p->x_md = put(n * p->max_md); p->x_mdlen = put(n * sizeof(uint32_t)); p->x_edits = put(4 * n * sizeof(uint32_t));
    p->x_btemp = align_up(x, 256);
    p->x_rec = 0;
    p->x_zout = 0;
    p->x_ztemp = align_up(std::max(p->rec_cap, p->z_cap), 256);

    char* fake = (char*)(uintptr_t)4096;                              // queries only: never dereferenced
    size_t tb = 0;
    int r = bam_map(p, fake, p->n_reads, nullptr, &tb, nullptr);
    if (r != NVB_E_TEMP_SIZE) return r == NVB_OK ? NVB_E_INVALID : r;
    p->map_temp = tb;
    tb = 0;
    r = bam_records(p, fake, p->n_reads, nullptr, &tb, nullptr);
    if (r != NVB_E_TEMP_SIZE) return r == NVB_OK ? NVB_E_INVALID : r;
    p->bam_temp = tb;
    p->z_temp = 0;
    if (p->bp.compress) {
        tb = 0;
        r = bam_compress(p, fake, p->n_reads, nullptr, &tb, nullptr);
        if (r != NVB_E_TEMP_SIZE) return r == NVB_OK ? NVB_E_INVALID : r;
        p->z_temp = tb;
    }
    size_t end = p->x_map + p->map_temp;
    end = std::max(end, p->x_btemp + p->bam_temp);
    if (p->bp.compress) end = std::max(end, p->x_ztemp + p->z_temp);
    p->slot_bytes = align_up(p->o_x + end, 256);
    return NVB_OK;
}

extern "C" int nvb_pipeline_create_bam(const nvb_fm_index* fmi, const uint32_t* d_genome, const nvb_seed_extend_params* params,
                                       const nvb_pair_params* pair_params, const nvb_pipeline_bam_params* bam,
                                       uint32_t max_reads, uint32_t read_len, uint32_t words_per_read, uint32_t read_bits,
                                       uint32_t hit_capacity, uint32_t depth, nvb_pipeline** out)
{
    if (!fmi || !d_genome || !params || !out || max_reads == 0 || depth == 0 || depth > 16) return NVB_E_INVALID;
    if (!(read_bits == 2 || read_bits == 4) || (uint64_t)words_per_read * (32u / read_bits) < read_len) return NVB_E_INVALID;
    if (pair_params && ((max_reads & 1u) || !valid_pair_policy(pair_params))) return NVB_E_INVALID;
    if (!bam || !bam->mapq || !bam->mapq->d_min_score || !bam->d_contig_begin || bam->n_contigs == 0 || bam->max_name_bytes == 0)
        return NVB_E_INVALID;
    if (params->d_read_quals || (params->scheme.d_qual_table && !bam->has_quals)) return NVB_E_INVALID;
    if (bam->mapq->max_read_len < read_len) return NVB_E_INVALID;
    if (read_len > 512u) return NVB_E_UNSUPPORTED;
    nvb_pipeline* p = new (std::nothrow) nvb_pipeline();
    if (!p) return (int)cudaErrorMemoryAllocation;
    *out = nullptr;
    p->fmi = *fmi; p->d_genome = d_genome; p->params = *params; p->paired = pair_params != nullptr;
    if (pair_params) p->pair = *pair_params;
    p->n_reads = max_reads; p->read_len = read_len; p->wpr = words_per_read; p->bits = read_bits; p->hit_capacity = hit_capacity; p->depth = depth;
    p->bam = true; p->bp = *bam; p->mapq = *bam->mapq; p->bp.mapq = &p->mapq;
    p->max_ops = bam->max_ops ? bam->max_ops : 2u * read_len + params->band_len;
    p->max_cigar = bam->max_cigar ? bam->max_cigar : p->max_ops + 2u;
    p->max_md = bam->max_md ? bam->max_md : 3u * p->max_ops + 1u;
    p->n_compute = 1;
    if (const char* e = getenv("NVB_PIPELINE_COMPUTE_STREAMS")) { const int v = atoi(e); if (v >= 1) p->n_compute = (uint32_t)v; }
    if (p->n_compute > depth) p->n_compute = depth;
    int rc = NVB_OK;
#define PIPE_TRY(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { rc = (int)_e; goto fail; } } while (0)
    {
        PIPE_TRY(cudaGetDevice(&p->device));
        rc = bam_layout(p);
        if (rc != NVB_OK) goto fail;
        PIPE_TRY(cudaStreamCreateWithFlags(&p->h2d, cudaStreamNonBlocking));
        PIPE_TRY(cudaStreamCreateWithFlags(&p->d2h, cudaStreamNonBlocking));
        PIPE_TRY(cudaStreamCreateWithFlags(&p->pay, cudaStreamNonBlocking));
        for (uint32_t i = 0; i < p->n_compute; ++i) PIPE_TRY(cudaStreamCreateWithFlags(&p->compute[i], cudaStreamNonBlocking));
        p->slots.resize(depth);
        p->bslots.resize(depth);
        uint32_t k = 0;
        for (uint32_t i = 0; i < depth; ++i) {
            nvb_pipeline::Slot& s = p->slots[i];
            p->bslots[i] = nvb_pipeline::BamSlot();
            s.out_bytes = sizeof(BamFixed); s.busy = false;
            s.compute = p->compute[k++ % p->n_compute];
            PIPE_TRY(cudaMalloc((void**)&s.d_in, p->slot_bytes));
            PIPE_TRY(cudaMemset(s.d_in, 0, p->o_x));
            s.d_out = (char*)s.d_in + p->o_fixed;
            PIPE_TRY(cudaHostAlloc((void**)&s.h_out, sizeof(BamFixed), cudaHostAllocDefault));
            PIPE_TRY(cudaMemset(s.d_out, 0, sizeof(BamFixed)));
            PIPE_TRY(cudaEventCreateWithFlags(&s.ev_in, cudaEventDisableTiming));
            PIPE_TRY(cudaEventCreate(&s.ev_start));
            PIPE_TRY(cudaEventCreate(&s.ev_done));
            PIPE_TRY(cudaEventCreateWithFlags(&s.ev_out, cudaEventDisableTiming));
            PIPE_TRY(cudaEventCreateWithFlags(&p->bslots[i].ev_pay, cudaEventDisableTiming));
        }
    }
#undef PIPE_TRY
    *out = p;
    return NVB_OK;
fail:
    nvb_pipeline_destroy(p);
    return rc;
}

// the payload of the slot's batch to its pinned host buffer, exactly its byte count; blocks until it is there
static int bam_fetch(nvb_pipeline* p, uint32_t k)
{
    nvb_pipeline::Slot& s = p->slots[k];
    nvb_pipeline::BamSlot& b = p->bslots[k];
    if (s.busy) NVB_CUDA_TRY(cudaEventSynchronize(s.ev_out));       // the counts are on the host
    s.busy = false;
    if (b.copied) return NVB_OK;
    const BamFixed* fx = (const BamFixed*)s.h_out;
    const size_t bytes = p->bp.compress ? fx->payload_z : fx->record_bytes;
    if (bytes > b.pay_cap) {
        if (b.h_pay) NVB_CUDA_TRY(cudaFreeHost(b.h_pay));
        b.h_pay = nullptr; b.pay_cap = 0;
        const size_t cap = align_up(bytes + bytes / 4, 1u << 20);
        NVB_CUDA_TRY(cudaHostAlloc((void**)&b.h_pay, cap, cudaHostAllocDefault));
        b.pay_cap = cap;
    }
    if (bytes) {
        const char* x = (const char*)s.d_in + p->o_x;
        NVB_CUDA_TRY(cudaMemcpyAsync(b.h_pay, x + (p->bp.compress ? p->x_zout : p->x_rec), bytes, cudaMemcpyDeviceToHost, p->pay));
        NVB_CUDA_TRY(cudaEventRecord(b.ev_pay, p->pay));
        NVB_CUDA_TRY(cudaEventSynchronize(b.ev_pay));
    }
    b.copied = true;
    return NVB_OK;
}

// the host-side checks of a submit (no CUDA call)
static bool bam_submit_ok(const nvb_pipeline_bam_params* bp, bool paired, uint32_t max_reads, uint32_t read_len, uint32_t n,
                          const uint32_t* h_read_words, const uint8_t* h_quals, const uint32_t* h_lengths, const char* h_names,
                          const uint32_t* h_name_offsets)
{
    if (!bp || !h_read_words || !h_names || !h_name_offsets) return false;
    if (n == 0 || n > max_reads || (paired && (n & 1u))) return false;
    if ((bp->has_quals && !h_quals) || (bp->has_lengths && !h_lengths)) return false;
    const uint32_t n_names = paired ? n / 2u : n;
    if (h_name_offsets[0] != 0u || h_name_offsets[n_names] > bp->max_name_bytes) return false;
    for (uint32_t j = 0; j < n_names; ++j) if (h_name_offsets[j + 1] <= h_name_offsets[j]) return false;
    if (bp->has_lengths) for (uint32_t i = 0; i < n; ++i) if (h_lengths[i] == 0u || h_lengths[i] > read_len) return false;
    return true;
}

extern "C" int nvb_debug_pipeline_bam_submit_check(const nvb_pipeline_bam_params* bam, uint32_t paired, uint32_t max_reads, uint32_t read_len,
                                                   uint32_t n_reads, const uint32_t* h_read_words, const uint8_t* h_quals,
                                                   const uint32_t* h_lengths, const char* h_names, const uint32_t* h_name_offsets)
{
    return bam_submit_ok(bam, paired != 0u, max_reads, read_len, n_reads, h_read_words, h_quals, h_lengths, h_names, h_name_offsets)
               ? NVB_OK : NVB_E_INVALID;
}

extern "C" int nvb_pipeline_submit_bam(nvb_pipeline* p, uint32_t n, const uint32_t* h_read_words, const uint8_t* h_quals,
                                       const uint32_t* h_lengths, const char* h_names, const uint32_t* h_name_offsets, uint32_t* ticket)
{
    if (!p || !p->bam || !ticket) return NVB_E_INVALID;
    if (!bam_submit_ok(&p->bp, p->paired, p->n_reads, p->read_len, n, h_read_words, h_quals, h_lengths, h_names, h_name_offsets))
        return NVB_E_INVALID;
    const uint32_t n_names = p->paired ? n / 2u : n;

    const uint32_t k = (uint32_t)(p->next % p->depth);
    nvb_pipeline::Slot& s = p->slots[k];
    nvb_pipeline::BamSlot& b = p->bslots[k];
    if (b.filled) { const int r = bam_fetch(p, k); if (r != NVB_OK) return r; }     // the slot's previous payload first
    char* base = (char*)s.d_in;
    // copy-in must not overwrite inputs that the slot's previous kernels may still be reading
    NVB_CUDA_TRY(cudaStreamWaitEvent(p->h2d, s.ev_done, 0));
    NVB_CUDA_TRY(cudaMemcpyAsync(base + p->o_words, h_read_words, (size_t)n * p->wpr * sizeof(uint32_t), cudaMemcpyHostToDevice, p->h2d));
    if (p->bp.has_quals)
        NVB_CUDA_TRY(cudaMemcpyAsync(base + p->o_quals, h_quals, (size_t)n * p->wpr * (32u / p->bits), cudaMemcpyHostToDevice, p->h2d));
    if (p->bp.has_lengths)
        NVB_CUDA_TRY(cudaMemcpyAsync(base + p->o_lens, h_lengths, (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice, p->h2d));
    NVB_CUDA_TRY(cudaMemcpyAsync(base + p->o_names, h_names, h_name_offsets[n_names], cudaMemcpyHostToDevice, p->h2d));
    NVB_CUDA_TRY(cudaMemcpyAsync(base + p->o_noff, h_name_offsets, ((size_t)n_names + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, p->h2d));
    NVB_CUDA_TRY(cudaEventRecord(s.ev_in, p->h2d));
    NVB_CUDA_TRY(cudaStreamWaitEvent(s.compute, s.ev_in, 0));
    NVB_CUDA_TRY(cudaStreamWaitEvent(s.compute, s.ev_out, 0));       // ... nor may the kernels overwrite counts still being copied out
    NVB_CUDA_TRY(cudaEventRecord(s.ev_start, s.compute));
    char* x = base + p->o_x;
    size_t tb = p->map_temp;
    int r = bam_map(p, base, n, x + p->x_map, &tb, s.compute);
    if (r != NVB_OK) return r;
    nvb_string_set rs = bam_reads(p, base);
    nvb_best_alignment_out ba = bam_alignment(p, base);
    nvb_finish_out fo = bam_finish_out(p, base);
    r = nvb_finish_alignments(p->d_genome, p->fmi.length, &rs, n, &ba, &fo, s.compute);
    if (r != NVB_OK) return r;
    tb = p->bam_temp;
    r = bam_records(p, base, n, x + p->x_btemp, &tb, s.compute);
    if (r != NVB_OK) return r;
    BamFixed* fx = (BamFixed*)(base + p->o_fixed);
    NVB_CUDA_TRY(cudaMemcpyAsync(&fx->record_bytes, base + p->o_recoff + (size_t)n * sizeof(uint64_t), sizeof(uint64_t),
                                 cudaMemcpyDeviceToDevice, s.compute));
    if (p->bp.compress) {
        tb = p->z_temp;
        r = bam_compress(p, base, n, x + p->x_ztemp, &tb, s.compute);
        if (r != NVB_OK) return r;
        NVB_CUDA_TRY(cudaMemcpyAsync(&fx->payload_z, base + p->o_zoff + (size_t)p->z_blocks * sizeof(uint64_t), sizeof(uint64_t),
                                     cudaMemcpyDeviceToDevice, s.compute));
    }
    NVB_CUDA_TRY(cudaEventRecord(s.ev_done, s.compute));
    NVB_CUDA_TRY(cudaStreamWaitEvent(p->d2h, s.ev_done, 0));
    NVB_CUDA_TRY(cudaMemcpyAsync(s.h_out, s.d_out, sizeof(BamFixed), cudaMemcpyDeviceToHost, p->d2h));
    NVB_CUDA_TRY(cudaEventRecord(s.ev_out, p->d2h));
    s.busy = true;
    b.n = n; b.filled = true; b.copied = false;
    *ticket = k;
    ++p->next;
    return NVB_OK;
}

extern "C" int nvb_pipeline_wait_bam(nvb_pipeline* p, uint32_t ticket, nvb_pipeline_bam_result* out)
{
    if (!p || !p->bam || ticket >= p->depth || !out) return NVB_E_INVALID;
    if (!p->bslots[ticket].filled) return NVB_E_INVALID;            // nothing was ever submitted to that slot
    const int rc = bam_fetch(p, ticket);                             // (waiting twice for the same ticket returns the same buffers)
    if (rc != NVB_OK) return rc;
    const nvb_pipeline::Slot& s = p->slots[ticket];
    const nvb_pipeline::BamSlot& b = p->bslots[ticket];
    const BamFixed* fx = (const BamFixed*)s.h_out;
    nvb_pipeline_bam_result r = {};
    r.payload = b.h_pay;
    r.record_bytes = fx->record_bytes;
    r.payload_bytes = p->bp.compress ? fx->payload_z : fx->record_bytes;
    r.n_records = fx->counts[0];
    r.n_blocks = p->bp.compress ? (uint32_t)((fx->record_bytes + 0xFEFFu) / 0xFF00u) : 0u;
    r.counts = fx->counts;
    r.n_hits = fx->n_hits;
    r.n_rescue = p->paired ? fx->n_rescue : nullptr;
    NVB_CUDA_TRY(cudaEventElapsedTime(&r.device_ms, s.ev_start, s.ev_done));
    *out = r;
    return NVB_OK;
}

extern "C" int nvb_debug_pipeline_bam_layout(const nvb_pipeline* p, uint64_t* out, uint32_t n_out)
{
    if (!p || !p->bam || !out) return NVB_E_INVALID;
    const uint64_t v[8] = {align_up((size_t)p->n_reads * p->max_ops, 256), p->rec_cap, p->x_fin, p->x_btemp, p->z_blocks, p->z_cap, p->o_x,
                           p->slot_bytes};
    for (uint32_t i = 0; i < n_out && i < 8; ++i) out[i] = v[i];
    return NVB_OK;
}

extern "C" size_t nvb_pipeline_slot_bytes(const nvb_pipeline* p)
{
    return p && p->bam ? p->slot_bytes : 0;
}
