/* nvbio_b200_debug.h -- test / tuning hooks exported by libnvbio_b200.so.  NOT part of the drop-in ABI (include/nvbio_b200.h):
 * they switch between the library's own GPU code paths so that the tests can exercise each of them and the microbenchmarks can
 * compare them; none of them changes a result.  Process-wide, not thread-safe. */
#ifndef NVBIO_B200_DEBUG_H
#define NVBIO_B200_DEBUG_H
#include <stdint.h>
#include "nvbio_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* banded / full-matrix Gotoh: 0 = automatic, 1 = the int32 one-alignment-per-thread kernels for everything */
void nvb_debug_force_gotoh_path(int path);
/* route of the last nvb_banded_gotoh_score(_indirect) / nvb_gotoh_score(_indirect) call (also the score pass inside the tracebacks):
 * *packed = 0 when no 16-bit packed kernel ran (the batch was refused by the admission rules or nvb_debug_force_gotoh_path(1)),
 * 1 = gotoh_pair_kernel / gotoh_full_pair_kernel, 2 = gotoh_full_warp_kernel; *n_int32 = the alignments that packed kernel put on the
 * int32 todo list (0 when *packed == 0).  Reads the caller's temp buffer of that call, so only while it is still allocated; synchronises
 * the device; changes no result */
int nvb_debug_gotoh_last_route(int* packed, uint32_t* n_int32);
/* full-matrix pair kernel occupancy variant: 0 = per-type default, 2 / 3 / 4 = minimum CTAs per SM */
void nvb_debug_full_minb(int minb);
/* full-matrix dispatch: 0 = by batch size, 1 = always the warp-per-pair kernel, 2 = never */
void nvb_debug_full_warp(int mode);
/* 1: nvb_gotoh_traceback runs the score dispatch, then the warp-per-alignment traceback of nvb_seed_extend_paired_traceback's rescued
   mates from those sinks (its slot pool and window cuts; pattern lengths up to 512, else NVB_E_UNSUPPORTED), and its temp query answers
   for that path; 0 (default): the one-alignment-per-thread direction-matrix kernel.  Same results; for tests of the warp kernel */
void nvb_debug_full_traceback_warp(int on);
/* 0: always the run-time-format pair kernel (PFMT 0); 1 (default): the compile-time 2- / 4-bit big-endian kernels where they apply */
void nvb_debug_pair_format(int on);
/* 1 (default): the banded pair kernels keep two pattern rows in flight per thread; 0: one row per loop iteration */
void nvb_debug_pair_rows2(int on);
/* 1 (default): nvb_banded_gotoh_traceback resolves gap-free alignments from the score kernels' sink (gapless fast path) and runs the
   direction-matrix traceback only for the others; 0: the direction-matrix traceback for every alignment */
void nvb_debug_traceback_fast(int on);
/* bytes of unused dynamic shared memory added to every banded pair-kernel CTA: measures what a landing buffer (e.g. for bulk
   copies of the text windows) would cost in resident CTAs per SM */
void nvb_debug_pair_extra_smem(int bytes);

/* seed + extend composition: 0 = automatic (the per-read path when no per-hit output is requested), 1 = always the per-hit path;
   any other value acts as 0 */
void nvb_debug_pipeline_path(int path);

/* seed-match stage of the per-read path with a k-mer table: 1 (default) = seeds on k-mers with three or more occurrences are finished
   by a second kernel, 0 = one pass.  Same results; for A/B timing and tests */
void nvb_debug_seed_split(int on);
/* *n = the number of seeds the first seed-match pass of the last two-pass call handed to the second (its todo lists).  Reads the
   caller's temp buffer of that call, so only while it is still allocated; synchronises the device */
int nvb_debug_seed_todo(uint32_t* n);

/* extension stage of the per-read path (LOCAL, constant scheme, 2-bit reads): 1 (default) = a job whose result the exact shortcut
   proves (the best segment of the seed's band diagonal beats every gapped alignment and every other diagonal) gets it without running
   the DP, 2 = the same without the one-gap check (only jobs whose segment beats every alignment with a gap), 0 = every job through the
   DP kernels.  Same results; for A/B timing and tests */
void nvb_debug_perfect_shortcut(int on);
/* *n = the number of alignment jobs the last per-read call with the exact shortcut left to the DP kernels.  Reads the caller's temp
   buffer of that call, so only while it is still allocated; synchronises the device */
int nvb_debug_dp_jobs(uint32_t* n);

/* the device build of the MAPQ function of nvb_seed_extend_mapq over n points (device arrays): d_mapq[i] = BowtieMapq2 of an unpaired
   read with best score d_best[i], a second score d_second[i] when d_has_second[i] != 0, perfect_score = d_len[i] * d_match_bonus[i],
   min_score = d_min_score[i] and the monotone branch when d_match_bonus[i] == 0.  For tests: it changes no state */
int nvb_debug_mapq_eval(const int32_t* d_best, const uint8_t* d_has_second, const int32_t* d_second, const uint32_t* d_len,
                        const int32_t* d_match_bonus, const int32_t* d_min_score, uint32_t n, uint8_t* d_mapq, void* stream);

/* nvb_bgzf_compress: CTAs of the resident compression grid, 0 (default) = one per SM.  Same output at every grid size; for tests */
void nvb_debug_bgzf_grid(uint32_t ctas);
/* nvb_bgzf_compress with its byte count in device memory, as the BAM mode of nvb_pipeline runs it: *d_n_bytes bytes at d_in (at most
   max_bytes; a larger value is taken as max_bytes).  max_bytes sizes the grids, the temp (the NVB_E_TEMP_SIZE answer) and the offsets:
   out->d_block_offsets has ceil(max_bytes / 0xFF00) + 1 entries, [0, n_blocks] as nvb_bgzf_compress writes them for the real count and
   the total repeated in every entry after n_blocks.  Members, offsets and capacity rules are otherwise those of nvb_bgzf_compress, byte
   for byte.  NVB_E_INVALID for a NULL d_n_bytes and nvb_bgzf_compress's checks on max_bytes.  For tests */
int nvb_debug_bgzf_compress_device_count(const uint8_t* d_in, const uint64_t* d_n_bytes, uint64_t max_bytes, const nvb_bgzf_out* out,
                                         void* d_temp, size_t* temp_bytes, void* stream);

/* the host-side checks nvb_pipeline_submit_bam makes before any CUDA call, for a pipeline made with `bam`, pair_params != NULL when
   paired != 0, max_reads and read_len: NVB_OK when a submit with these arguments passes them, else NVB_E_INVALID.  Needs no device;
   for tests of the rules without a pipeline */
int nvb_debug_pipeline_bam_submit_check(const nvb_pipeline_bam_params* bam, uint32_t paired, uint32_t max_reads, uint32_t read_len,
                                        uint32_t n_reads, const uint32_t* h_read_words, const uint8_t* h_quals, const uint32_t* h_lengths,
                                        const char* h_names, const uint32_t* h_name_offsets);
/* the slot layout of a BAM-mode pipeline, in bytes (see nvb_pipeline_create_bam): out[0] = O (the traceback ops), out[1] = R (the record
   bound), out[2] = the finish outputs' offset in the stage region (max(O, R)), out[3] = the records' temp offset, out[4] = BGZF blocks of
   R, out[5] = the BGZF members' capacity, out[6] = the stage region's offset in the slot, out[7] = slot bytes.  Writes min(n_out, 8)
   entries; NVB_E_INVALID for a NULL argument or a pipeline not in BAM mode.  For tests */
int nvb_debug_pipeline_bam_layout(const nvb_pipeline* p, uint64_t* out, uint32_t n_out);

#ifdef __cplusplus
}
#endif
#endif
