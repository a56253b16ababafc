"""ctypes loader for the in-tree CUDA library.  There is NO fallback: if the library is missing or
does not load, every entry point raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NVBIO_B200_LIB") or os.path.join(_HERE, "libnvbio_b200.so")     # (the override is for A/B experiments on kernels)

EXPORTS = [
    "nvb_version", "nvb_error_string",
    "nvb_fm_rank", "nvb_fm_rank4", "nvb_fm_match", "nvb_fm_match_approx", "nvb_fm_locate", "nvb_fm_filter_rank", "nvb_fm_filter_locate",
    "nvb_banded_gotoh_score", "nvb_banded_gotoh_score_indirect", "nvb_banded_gotoh_traceback", "nvb_gotoh_score", "nvb_gotoh_score_indirect", "nvb_banded_gotoh_score_window", "nvb_banded_gotoh_score_best2", "nvb_gotoh_traceback", "nvb_seed_extend_paired",
    "nvb_fm_build_occ", "nvb_fm_build_bwt", "nvb_fm_build_ktab", "nvb_fm_build_ktab_located", "nvb_fm_build_ktab_context", "nvb_fm_build_ktab_wide", "nvb_fm_build_rows", "nvb_seed_extend", "nvb_seed_extend_traceback", "nvb_seed_extend_mapq", "nvb_seed_extend_reseed", "nvb_seed_extend_all", "nvb_seed_extend_paired_mapq", "nvb_seed_extend_paired_traceback", "nvb_seed_extend_paired_reseed",
    "nvb_seed_extend_stage_ms",
    "nvb_dict_rank", "nvb_dict_rank4", "nvb_dict_build_occ",
    "nvb_map_seeds", "nvb_fm_locate_init", "nvb_fm_locate_lookup", "nvb_fm_locate_sorted",
    "nvb_pipeline_create", "nvb_pipeline_submit", "nvb_pipeline_wait", "nvb_pipeline_traffic", "nvb_pipeline_destroy",
    "nvb_pipeline_create_bam", "nvb_pipeline_submit_bam", "nvb_pipeline_wait_bam", "nvb_pipeline_slot_bytes",
    "nvb_finish_alignments", "nvb_bam_records", "nvb_bam_records_all", "nvb_bgzf_compress", "nvb_bam_sort", "nvb_bam_index", "nvb_sam_format",
]
# test / tuning hooks of include/nvbio_b200_debug.h (not part of the drop-in ABI)
DEBUG_EXPORTS = [
    "nvb_debug_gotoh_last_route", "nvb_debug_force_gotoh_path", "nvb_debug_full_minb", "nvb_debug_full_warp", "nvb_debug_full_traceback_warp",
    "nvb_debug_pair_format", "nvb_debug_pair_rows2", "nvb_debug_traceback_fast", "nvb_debug_pair_extra_smem",
    "nvb_debug_pipeline_path", "nvb_debug_seed_split", "nvb_debug_seed_todo", "nvb_debug_perfect_shortcut", "nvb_debug_dp_jobs", "nvb_debug_mapq_eval",
    "nvb_debug_bgzf_grid", "nvb_debug_bgzf_compress_device_count", "nvb_debug_pipeline_bam_submit_check",
    "nvb_debug_pipeline_bam_layout",
]


class NvbError(RuntimeError):
    pass


class FmIndexStruct(C.Structure):          # nvb_fm_index
    _fields_ = [("d_bwt_occ", C.c_void_p), ("d_ssa", C.c_void_p), ("length", C.c_uint32),
                ("primary", C.c_uint32), ("L2", C.c_uint32 * 5), ("sa_interval", C.c_uint32),
                ("d_ktab", C.c_void_p), ("ktab_k", C.c_uint32), ("ktab_located", C.c_uint32), ("d_rows", C.c_void_p)]


class StringSetStruct(C.Structure):        # nvb_string_set
    _fields_ = [("d_words", C.c_void_p), ("bits", C.c_uint32), ("big_endian", C.c_uint32),
                ("d_offsets", C.c_void_p), ("d_lengths", C.c_void_p), ("stride", C.c_uint32),
                ("length", C.c_uint32)]


class GotohSchemeStruct(C.Structure):      # nvb_gotoh_scheme
    _fields_ = [("match", C.c_int32), ("mismatch", C.c_int32), ("pattern_gap_open", C.c_int32),
                ("pattern_gap_ext", C.c_int32), ("text_gap_open", C.c_int32), ("text_gap_ext", C.c_int32),
                ("d_qual_table", C.c_void_p), ("qual_table_min", C.c_int32), ("qual_table_max", C.c_int32)]


class SeedExtendParamsStruct(C.Structure):  # nvb_seed_extend_params
    _fields_ = [("seed_len", C.c_uint32), ("seed_interval", C.c_uint32), ("band_len", C.c_uint32),
                ("type", C.c_uint32), ("both_strands", C.c_uint32), ("max_seed_hits", C.c_uint32),
                ("dedup_jobs", C.c_uint32), ("scheme", GotohSchemeStruct), ("d_read_quals", C.c_void_p)]


class BestAlignmentOutStruct(C.Structure):   # nvb_best_alignment_out
    _fields_ = [("d_ops", C.c_void_p), ("max_ops", C.c_uint32), ("d_n_ops", C.c_void_p), ("d_begin", C.c_void_p),
                ("d_strand", C.c_void_p)]


class FinishOutStruct(C.Structure):        # nvb_finish_out
    _fields_ = [("d_cigar", C.c_void_p), ("max_cigar", C.c_uint32), ("d_n_cigar", C.c_void_p), ("d_md", C.c_void_p), ("max_md", C.c_uint32),
                ("d_md_len", C.c_void_p), ("d_edits", C.c_void_p)]


class BamInStruct(C.Structure):           # nvb_bam_in
    _fields_ = [("reads", StringSetStruct), ("d_read_quals", C.c_void_p), ("d_n_ops", C.c_void_p), ("d_begin", C.c_void_p),
                ("d_strand", C.c_void_p), ("finish", FinishOutStruct), ("d_score", C.c_void_p), ("d_mapq", C.c_void_p),
                ("d_second_score", C.c_void_p), ("d_pair_flags", C.c_void_p), ("d_contig_begin", C.c_void_p), ("n_contigs", C.c_uint32),
                ("d_names", C.c_void_p), ("d_name_offsets", C.c_void_p)]


class BamAllInStruct(C.Structure):        # nvb_bam_all_in
    _fields_ = [("base", BamInStruct), ("d_first", C.c_void_p), ("capacity", C.c_uint32)]


class BamOutStruct(C.Structure):          # nvb_bam_out
    _fields_ = [("d_records", C.c_void_p), ("capacity", C.c_uint64), ("d_offsets", C.c_void_p), ("d_counts", C.c_void_p)]


class BgzfOutStruct(C.Structure):         # nvb_bgzf_out
    _fields_ = [("d_out", C.c_void_p), ("capacity", C.c_uint64), ("d_block_offsets", C.c_void_p)]


class BamSortOutStruct(C.Structure):      # nvb_bam_sort_out
    _fields_ = [("d_records", C.c_void_p), ("capacity", C.c_uint64), ("d_offsets", C.c_void_p), ("d_order", C.c_void_p)]


class BaiOutStruct(C.Structure):          # nvb_bai_out
    _fields_ = [("d_bai", C.c_void_p), ("capacity", C.c_uint64), ("d_size", C.c_void_p), ("d_status", C.c_void_p)]


class SamOutStruct(C.Structure):          # nvb_sam_out
    _fields_ = [("d_text", C.c_void_p), ("capacity", C.c_uint64), ("d_offsets", C.c_void_p), ("d_rejected", C.c_void_p)]


class MapqParamsStruct(C.Structure):       # nvb_mapq_params
    _fields_ = [("d_min_score", C.c_void_p), ("max_read_len", C.c_uint32), ("match_bonus", C.c_int32)]


class MapqOutStruct(C.Structure):          # nvb_mapq_out
    _fields_ = [("d_second_score", C.c_void_p), ("d_second_pos", C.c_void_p), ("d_second_strand", C.c_void_p), ("d_mapq", C.c_void_p)]


class ReseedParamsStruct(C.Structure):      # nvb_reseed_params
    _fields_ = [("max_reseed", C.c_uint32), ("rep_seeds", C.c_uint32), ("d_min_score", C.c_void_p), ("max_read_len", C.c_uint32)]


class ReseedOutStruct(C.Structure):         # nvb_reseed_out
    _fields_ = [("d_rounds", C.c_void_p), ("d_active", C.c_void_p)]


class AllParamsStruct(C.Structure):         # nvb_all_params
    _fields_ = [("max_per_read", C.c_uint32), ("capacity", C.c_uint32)]


class AllOutStruct(C.Structure):            # nvb_all_out
    _fields_ = [("d_first", C.c_void_p), ("d_read", C.c_void_p), ("d_score", C.c_void_p), ("d_pos", C.c_void_p),
                ("alignment", BestAlignmentOutStruct), ("d_count", C.c_void_p)]


class PairParamsStruct(C.Structure):        # nvb_pair_params
    _fields_ = [("min_frag", C.c_uint32), ("max_frag", C.c_uint32), ("min_mate_score", C.c_int32), ("rescue_capacity", C.c_uint32),
                ("policy", C.c_uint32), ("flags", C.c_uint32)]


class PairOutStruct(C.Structure):           # nvb_pair_out
    _fields_ = [("d_pair_score", C.c_void_p), ("d_pair_flags", C.c_void_p), ("d_mate_score", C.c_void_p), ("d_mate_pos", C.c_void_p),
                ("d_mate_strand", C.c_void_p), ("d_n_rescue", C.c_void_p)]


class PairMapqOutStruct(C.Structure):       # nvb_pair_mapq_out
    _fields_ = [("d_second_pair_score", C.c_void_p), ("d_second_mate_pos", C.c_void_p), ("d_second_mate_strand", C.c_void_p),
                ("d_mate_second_score", C.c_void_p), ("d_mate_mapq", C.c_void_p)]


class PipelineResultStruct(C.Structure):    # nvb_pipeline_result
    _fields_ = [("best_score", C.c_void_p), ("best_pos", C.c_void_p), ("n_hits", C.c_void_p), ("pair_score", C.c_void_p),
                ("pair_flags", C.c_void_p), ("mate_score", C.c_void_p), ("mate_pos", C.c_void_p), ("mate_strand", C.c_void_p),
                ("n_rescue", C.c_void_p), ("device_ms", C.c_float)]


class PipelineBamParamsStruct(C.Structure):  # nvb_pipeline_bam_params
    _fields_ = [("mapq", C.c_void_p), ("d_contig_begin", C.c_void_p), ("n_contigs", C.c_uint32), ("max_name_bytes", C.c_uint32),
                ("has_quals", C.c_uint32), ("has_lengths", C.c_uint32), ("compress", C.c_uint32), ("max_ops", C.c_uint32),
                ("max_cigar", C.c_uint32), ("max_md", C.c_uint32)]


class PipelineBamResultStruct(C.Structure):  # nvb_pipeline_bam_result
    _fields_ = [("payload", C.c_void_p), ("payload_bytes", C.c_uint64), ("record_bytes", C.c_uint64), ("n_records", C.c_uint32),
                ("n_blocks", C.c_uint32), ("counts", C.c_void_p), ("n_hits", C.c_void_p), ("n_rescue", C.c_void_p), ("device_ms", C.c_float)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NvbError("nvbio_b200: %s is missing -- run `python -m nvbio_b200.build` "
                           "(there is no CPU fallback)" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        _lib.nvb_error_string.restype = C.c_char_p
        _lib.nvb_pipeline_destroy.restype = None
        _lib.nvb_pipeline_traffic.restype = None
        _lib.nvb_pipeline_slot_bytes.restype = C.c_size_t
        for name in EXPORTS + DEBUG_EXPORTS:
            getattr(_lib, name)            # raises AttributeError if a symbol is not exported
    return _lib


def check(err, what=""):
    if err != 0:
        msg = lib().nvb_error_string(C.c_int(err)).decode()
        raise NvbError("%s failed: %s (%d)" % (what or "nvbio_b200 call", msg, err))
