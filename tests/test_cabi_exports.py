"""CPU: the C-ABI library builds, loads, and exports every symbol include/nvbio_b200.h declares."""
import ctypes as C
import os
import re
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols(header="nvbio_b200.h"):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nvb_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_everything():
    from nvbio_b200 import build
    path = build.build()
    assert os.path.exists(path)
    lib = C.CDLL(path)
    names = declared_symbols()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
    lib.nvb_version.restype = C.c_int
    assert lib.nvb_version() == 100
    lib.nvb_error_string.restype = C.c_char_p
    assert b"invalid" in lib.nvb_error_string(C.c_int(-1))


def test_python_mirror_lists_same_exports():
    from nvbio_b200 import _lib
    assert set(_lib.EXPORTS) == set(declared_symbols())
    # the test / tuning hooks: listed apart, and every one of them exported (lib() resolves both lists)
    assert set(_lib.DEBUG_EXPORTS) == set(declared_symbols("nvbio_b200_debug.h"))
    L = _lib.lib()
    for n in _lib.DEBUG_EXPORTS:
        assert hasattr(L, n), "missing export %s" % n


def test_argument_validation_without_gpu():
    """invalid arguments are rejected before any CUDA call"""
    from nvbio_b200 import _lib
    L = _lib.lib()
    assert L.nvb_fm_match(None, None, C.c_uint32(1), C.c_uint32(0), None, None) == -1
    tb = C.c_size_t(0)
    assert L.nvb_banded_gotoh_score(C.c_int(4), C.c_int(1), None, None, None, None, C.c_uint32(1), None, None, None, C.byref(tb), None) == -1


def test_argument_validation_of_the_widened_api():
    """full-matrix score / traceback, windowed score, the seed + extend traceback and the paired-end composition reject bad arguments
    with NVB_E_INVALID (-1) or NVB_E_UNSUPPORTED (-4) before any CUDA call; size queries answer NVB_E_TEMP_SIZE (-2) without touching the
    device"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, PairParamsStruct, PairOutStruct, SeedExtendParamsStruct, FmIndexStruct,
                                 BestAlignmentOutStruct)
    L = _lib.lib()
    tb = C.c_size_t(0)
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
    tt = StringSetStruct(); tt.d_words = 16; tt.bits = 2; tt.big_endian = 1; tt.stride = 512; tt.length = 500
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    # type out of range / NULL scheme
    assert L.nvb_gotoh_score(C.c_int(3), C.byref(sch), C.byref(ss), None, C.byref(tt), C.c_uint32(4), None, None, None, C.byref(tb), None) == -1
    assert L.nvb_gotoh_score(C.c_int(1), None, C.byref(ss), None, C.byref(tt), C.c_uint32(4), None, None, None, C.byref(tb), None) == -1
    # size query: 8 B x (n + 1) x max text length for patterns longer than one stripe (+ the todo list)
    assert L.nvb_gotoh_score(C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(tt), C.c_uint32(1000), None, None, None, C.byref(tb), None) == -2
    assert tb.value >= 8 * 1001 * 500
    big = StringSetStruct(); big.d_words = 16; big.bits = 2; big.big_endian = 1; big.stride = 70000; big.length = 70000
    assert L.nvb_gotoh_score(C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(big), C.c_uint32(4), None, None, None, C.byref(tb), None) == -4
    assert L.nvb_gotoh_score_indirect(C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(tt), None, C.c_uint32(4), None, None, None, C.byref(tb), None) == -1
    tb2 = C.c_size_t(0)
    assert L.nvb_gotoh_traceback(C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(tt), C.c_uint32(10), None, None, None, None, C.c_uint32(700), None,
                                 None, C.byref(tb2), None) == -2
    assert tb2.value >= 10 * 500 * (5 * 16 + 8)          # direction matrix + boundary column
    # windowed: empty window, unknown band
    assert L.nvb_banded_gotoh_score_window(C.c_int(31), C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(tt), C.c_uint32(4),
                                           C.c_uint32(32), C.c_uint32(32), None, None, None, None, None, None) == -1
    assert L.nvb_banded_gotoh_score_window(C.c_int(9), C.c_int(1), C.byref(sch), C.byref(ss), None, C.byref(tt), C.c_uint32(4),
                                           C.c_uint32(0), C.c_uint32(32), None, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), None) == -1
    # paired: missing outputs, single-strand parameters
    pp = PairParamsStruct(); pp.min_frag, pp.max_frag, pp.min_mate_score, pp.rescue_capacity = 0, 500, 50, 100
    po = PairOutStruct()
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    assert L.nvb_seed_extend_paired(C.byref(fm), C.c_void_p(16), C.byref(ss), C.c_uint32(8), C.byref(sp), C.c_uint32(100), C.byref(pp), C.byref(po),
                                    None, None, C.byref(tb), None) == -1
    for f in ("d_pair_score", "d_pair_flags", "d_mate_score", "d_mate_pos", "d_mate_strand"):
        setattr(po, f, 16)
    sp.both_strands = 0
    assert L.nvb_seed_extend_paired(C.byref(fm), C.c_void_p(16), C.byref(ss), C.c_uint32(8), C.byref(sp), C.c_uint32(100), C.byref(pp), C.byref(po),
                                    None, None, C.byref(tb), None) == -1
    sp.both_strands = 1
    pp.min_frag = 600
    assert L.nvb_seed_extend_paired(C.byref(fm), C.c_void_p(16), C.byref(ss), C.c_uint32(8), C.byref(sp), C.c_uint32(100), C.byref(pp), C.byref(po),
                                    None, None, C.byref(tb), None) == -1
    pp.min_frag = 0
    # 8-bit reads are NVB_E_UNSUPPORTED (-4); a failed check of the pair arguments, outputs or parameters wins over it
    s8 = StringSetStruct(); s8.d_words = 16; s8.bits = 8; s8.big_endian = 1; s8.stride = 152; s8.length = 150
    r = lambda x: C.byref(x) if x is not None else None      # noqa: E731

    def paired(reads=s8, pp_=pp, po_=po, temp_bytes=tb, n_pairs=8):
        return L.nvb_seed_extend_paired(C.byref(fm), C.c_void_p(16), r(reads), C.c_uint32(n_pairs), C.byref(sp), C.c_uint32(100), r(pp_), r(po_),
                                        None, None, r(temp_bytes), None)
    assert paired() == -4
    assert paired(pp_=None) == -1 and paired(po_=None) == -1 and paired(temp_bytes=None) == -1 and paired(n_pairs=0x40000000) == -1
    assert paired(reads=None) == -1 and paired(reads=ss, temp_bytes=None) == -1 and paired(reads=ss, n_pairs=0x40000000) == -1
    po.d_mate_pos = None
    assert paired() == -1
    po.d_mate_pos = 16
    pp.max_frag = 0
    assert paired() == -1
    pp.max_frag = 500

    # single-end traceback: NULL or incomplete best_alignment (-1), also with 8-bit reads
    def traceback(ba, reads=s8):
        return L.nvb_seed_extend_traceback(C.byref(fm), C.c_void_p(16), r(reads), C.c_uint32(8), C.byref(sp), C.c_uint32(100), C.c_void_p(16),
                                           C.c_void_p(16), None, None, None, None, None, r(ba), None, C.byref(tb), None)
    assert traceback(None) == -1 and traceback(None, reads=ss) == -1
    for k in ("d_ops", "d_n_ops", "d_begin", "max_ops"):
        ba = BestAlignmentOutStruct(); ba.d_ops = 16; ba.max_ops = 300; ba.d_n_ops = 16; ba.d_begin = 16
        setattr(ba, k, None if k != "max_ops" else 0)
        assert traceback(ba) == -1 and traceback(ba, reads=ss) == -1, k
    ba = BestAlignmentOutStruct(); ba.d_ops = 16; ba.max_ops = 300; ba.d_n_ops = 16; ba.d_begin = 16
    assert traceback(ba) == -4 and traceback(ba, reads=None) == -1


def test_no_oracle_in_product():
    """the product package must not import / link the oracle"""
    pkg = os.path.join(ROOT, "nvbio_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "oracle" not in txt.lower() or f == "synth.py", (f, "mentions the oracle")
