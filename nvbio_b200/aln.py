"""Host-side mirror of nvbio::aln for the banded Gotoh scoring path (nvbio/alignment/alignment_base.h,
utils.h, batched.h) over the C ABI."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional, Tuple
import numpy as np
import torch
from ._lib import lib, check, GotohSchemeStruct
from .strings import PackedStringSet

GLOBAL, LOCAL, SEMI_GLOBAL = 0, 1, 2        # aln::AlignmentType (alignment_base.h:54)


@dataclass
class SimpleGotohScheme:
    """aln::SimpleGotohScheme(match, mismatch, gap_open, gap_ext) (nvbio/alignment/utils.h:114-135)"""
    match: int
    mismatch: int
    gap_open: int
    gap_ext: int

    def struct(self) -> GotohSchemeStruct:
        s = GotohSchemeStruct()
        s.match, s.mismatch = self.match, self.mismatch
        s.pattern_gap_open = s.text_gap_open = self.gap_open
        s.pattern_gap_ext = s.text_gap_ext = self.gap_ext
        s.d_qual_table = None
        s.qual_table_min = s.qual_table_max = 0
        return s


class QualityGotohScheme:
    """nvBowtie's SmithWatermanScoringScheme<QualCost,ConstantCost> seen through the Gotoh interface
    (nvBowtie/bowtie2/cuda/scoring.h:203-317): substitution = r==q ? match(q) : -mmp(q).  The float
    expression of QualCost (scoring.h:96-100) is evaluated HERE, on the host, in float32 exactly as
    written, and shipped as a 256x2 int32 table."""

    @staticmethod
    def host_table(match_bonus: int, mm_min: int, mm_max: int) -> np.ndarray:
        """[256, 2] int32: (substitution on a match, on a mismatch) per base quality -- QualCost::operator() (scoring.h:96-100:
        min + int(float(min(q,40) / 40.0f) * (max - min))) in float32, truncated towards zero like the C cast"""
        q = np.arange(256)
        frac = (np.minimum(q, 40).astype(np.float32) / np.float32(40.0)).astype(np.float32)
        mmp = mm_min + np.trunc(frac * np.float32(mm_max - mm_min)).astype(np.int32)
        return np.ascontiguousarray(np.stack([np.full(256, match_bonus, dtype=np.int32), (-mmp).astype(np.int32)], axis=1))

    def __init__(self, match_bonus: int, mm_min: int, mm_max: int, read_gap_const: int, read_gap_coeff: int,
                 ref_gap_const: int, ref_gap_coeff: int, device="cuda"):
        tab = self.host_table(match_bonus, mm_min, mm_max)
        self.table_host = np.ascontiguousarray(tab)
        self.table = torch.from_numpy(self.table_host).to(device)
        self.pgo, self.pge = -read_gap_const - read_gap_coeff, -read_gap_coeff
        self.tgo, self.tge = -ref_gap_const - ref_gap_coeff, -ref_gap_coeff
        self.match_bonus = match_bonus

    def struct(self) -> GotohSchemeStruct:
        s = GotohSchemeStruct()
        s.match, s.mismatch = self.match_bonus, int(self.table_host[0, 1])
        s.pattern_gap_open, s.pattern_gap_ext = self.pgo, self.pge
        s.text_gap_open, s.text_gap_ext = self.tgo, self.tge
        s.d_qual_table = self.table.data_ptr()
        s.qual_table_min, s.qual_table_max = int(self.table_host.min()), int(self.table_host.max())
        return s


@dataclass
class GotohAligner:
    """aln::GotohAligner<TYPE, scheme> / make_gotoh_aligner<TYPE>(scheme) (alignment_base.h:255-298)"""
    type: int
    scheme: object


def make_gotoh_aligner(type: int, scheme) -> GotohAligner:
    return GotohAligner(type, scheme)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def batch_banded_alignment_score(band_len: int, aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet,
                                 quals: Optional[torch.Tensor] = None,
                                 out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                                 temp: Optional[torch.Tensor] = None):
    """aln::batch_banded_alignment_score<BAND_LEN>(aligner, patterns, texts, sinks, DeviceThreadScheduler(), ...)
    (nvbio/alignment/batched_inl.h:1067-1101).  Returns (scores int32[n], sinks int32[n,2]) = BestSink<int32>."""
    L = lib()
    n = patterns.count
    assert texts.count == n
    dev = patterns.words.device
    if out is None:
        out = (torch.empty(n, dtype=torch.int32, device=dev), torch.empty((n, 2), dtype=torch.int32, device=dev))
    score, sink = out
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    qp = C.c_void_p(quals.data_ptr()) if quals is not None else None
    tb = C.c_size_t(0 if temp is None else temp.numel())
    if temp is None:
        r = L.nvb_banded_gotoh_score(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p), qp, C.byref(t),
                                     C.c_uint32(n), C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()),
                                     None, C.byref(tb), _stream())
        if r != -2:
            check(r, "nvb_banded_gotoh_score(size query)")
        temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(L.nvb_banded_gotoh_score(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p), qp, C.byref(t),
                                   C.c_uint32(n), C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()),
                                   C.c_void_p(temp.data_ptr()), C.byref(tb), _stream()), "nvb_banded_gotoh_score")
    return score, sink


def banded_temp_bytes(band_len, aligner, patterns, texts) -> int:
    L = lib()
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    tb = C.c_size_t(0)
    r = L.nvb_banded_gotoh_score(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p), None, C.byref(t),
                                 C.c_uint32(patterns.count), None, None, None, C.byref(tb), _stream())
    if r not in (0, -2):
        check(r, "nvb_banded_gotoh_score(size query)")
    return int(tb.value)


def batch_banded_alignment_traceback(band_len: int, aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet,
                                     quals: Optional[torch.Tensor] = None, max_ops: Optional[int] = None):
    """aln::banded_alignment_traceback<BAND_LEN,...> for a batch (nvbio/alignment/banded_inl.h:352-489).
    Returns dict(score[n], sink[n,2], source[n,2], ops[n,max_ops] uint8 in END->START push order (0 M, 1 I, 2 D), n_ops[n])."""
    L = lib()
    n = patterns.count
    dev = patterns.words.device
    if max_ops is None:
        max_ops = 2 * patterns.length + band_len           # every row (M / I) and every column (M / D) of the band: never truncated
    out = dict(score=torch.empty(n, dtype=torch.int32, device=dev), sink=torch.empty((n, 2), dtype=torch.int32, device=dev),
               source=torch.empty((n, 2), dtype=torch.int32, device=dev), ops=torch.zeros((n, max_ops), dtype=torch.uint8, device=dev),
               n_ops=torch.empty(n, dtype=torch.int32, device=dev))
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    qp = C.c_void_p(quals.data_ptr()) if quals is not None else None
    tb = C.c_size_t(0)

    def call(temp_ptr):
        return L.nvb_banded_gotoh_traceback(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p), qp, C.byref(t), C.c_uint32(n),
                                            C.c_void_p(out["score"].data_ptr()), C.c_void_p(out["sink"].data_ptr()),
                                            C.c_void_p(out["source"].data_ptr()), C.c_void_p(out["ops"].data_ptr()), C.c_uint32(max_ops),
                                            C.c_void_p(out["n_ops"].data_ptr()), temp_ptr, C.byref(tb), _stream())
    r = call(None)
    if r != -2:
        check(r, "nvb_banded_gotoh_traceback(size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(call(C.c_void_p(temp.data_ptr())), "nvb_banded_gotoh_traceback")
    return out


def cigar(ops_row, n_ops: int) -> str:
    """run-length CIGAR in START->END order from one row of END->START ops"""
    letters = "MID"
    seq = [int(v) for v in ops_row[:n_ops]][::-1]
    out, prev, cnt = [], None, 0
    for o in seq:
        if o == prev:
            cnt += 1
        else:
            if prev is not None:
                out.append("%d%s" % (cnt, letters[prev]))
            prev, cnt = o, 1
    if prev is not None:
        out.append("%d%s" % (cnt, letters[prev]))
    return "".join(out)


def batch_alignment_score(aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet, quals: Optional[torch.Tensor] = None):
    """aln::batch_alignment_score(aligner, patterns, texts, sinks, DeviceThreadScheduler(), ...) with a Gotoh aligner: the
    full-matrix DP of every pattern against its whole text (nvbio/alignment/batched_inl.h:984-1040).
    Returns (scores int32[n], sinks int32[n,2] = (text end, pattern end))."""
    L = lib()
    n = patterns.count
    dev = patterns.words.device
    score = torch.empty(n, dtype=torch.int32, device=dev)
    sink = torch.empty((n, 2), dtype=torch.int32, device=dev)
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    tb = C.c_size_t(0)

    def call(temp_ptr):
        return L.nvb_gotoh_score(C.c_int(aligner.type), C.byref(sch), C.byref(p), C.c_void_p(quals.data_ptr()) if quals is not None else None,
                                 C.byref(t), C.c_uint32(n),
                                 C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()), temp_ptr, C.byref(tb), _stream())
    r = call(None)
    if r != -2:
        check(r, "nvb_gotoh_score(size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(call(C.c_void_p(temp.data_ptr())), "nvb_gotoh_score")
    return score, sink


def batch_alignment_traceback(aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet, max_ops: Optional[int] = None,
                              quals: Optional[torch.Tensor] = None):
    """aln::alignment_traceback (full-matrix Gotoh) for a batch (nvbio/alignment/alignment_inl.h:365-530, batched_inl.h:607-860).
    Returns dict(score[n], sink[n,2], source[n,2], ops[n,max_ops] uint8 in END->START push order (0 M, 1 I, 2 D), n_ops[n])."""
    L = lib()
    n = patterns.count
    dev = patterns.words.device
    if max_ops is None:
        max_ops = patterns.length + texts.length + 1
    out = dict(score=torch.empty(n, dtype=torch.int32, device=dev), sink=torch.empty((n, 2), dtype=torch.int32, device=dev),
               source=torch.empty((n, 2), dtype=torch.int32, device=dev), ops=torch.zeros((n, max_ops), dtype=torch.uint8, device=dev),
               n_ops=torch.empty(n, dtype=torch.int32, device=dev))
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    tb = C.c_size_t(0)

    def call(temp_ptr):
        return L.nvb_gotoh_traceback(C.c_int(aligner.type), C.byref(sch), C.byref(p), C.c_void_p(quals.data_ptr()) if quals is not None else None,
                                     C.byref(t), C.c_uint32(n),
                                     C.c_void_p(out["score"].data_ptr()), C.c_void_p(out["sink"].data_ptr()),
                                     C.c_void_p(out["source"].data_ptr()), C.c_void_p(out["ops"].data_ptr()), C.c_uint32(max_ops),
                                     C.c_void_p(out["n_ops"].data_ptr()), temp_ptr, C.byref(tb), _stream())
    r = call(None)
    if r != -2:
        check(r, "nvb_gotoh_traceback(size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(call(C.c_void_p(temp.data_ptr())), "nvb_gotoh_traceback")
    return out


class BandedWindowState:
    """device state of a batch scored window by window (checkpoint bands, BestSinks, alive flags)"""

    def __init__(self, n: int, band_len: int, device):
        self.ckpt = torch.zeros((n, band_len, 2), dtype=torch.int16, device=device)
        self.score = torch.empty(n, dtype=torch.int32, device=device)
        self.sink = torch.empty((n, 2), dtype=torch.int32, device=device)
        self.alive = torch.empty(n, dtype=torch.uint8, device=device)


def batch_banded_alignment_score_window(band_len: int, aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet,
                                        window_begin: int, window_end: int, state: BandedWindowState,
                                        min_score: Optional[torch.Tensor] = None, quals: Optional[torch.Tensor] = None):
    """one [window_begin, window_end) pass of aln::banded_alignment_score<BAND_LEN>(..., window_begin, window_end, sink, checkpoint)
    over a batch (nvbio/alignment/banded_inl.h:178-218); call with consecutive windows, starting at 0"""
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    check(lib().nvb_banded_gotoh_score_window(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p),
                                              C.c_void_p(quals.data_ptr()) if quals is not None else None, C.byref(t), C.c_uint32(patterns.count),
                                              C.c_uint32(window_begin), C.c_uint32(window_end),
                                              C.c_void_p(min_score.data_ptr()) if min_score is not None else None,
                                              C.c_void_p(state.ckpt.data_ptr()), C.c_void_p(state.score.data_ptr()),
                                              C.c_void_p(state.sink.data_ptr()), C.c_void_p(state.alive.data_ptr()), _stream()),
          "nvb_banded_gotoh_score_window")
    return state


def batch_banded_alignment_score_best2(band_len: int, aligner: GotohAligner, patterns: PackedStringSet, texts: PackedStringSet, distinct_dist: int = 0,
                                       quals: Optional[torch.Tensor] = None) -> torch.Tensor:
    """banded Gotoh score into aln::Best2Sink<int32>(distinct_dist) (sink.h:114-147): int32 [n, 6] = (score1, sink1.x, sink1.y, score2, sink2.x, sink2.y)"""
    n = patterns.count
    out = torch.empty((n, 6), dtype=torch.int32, device=patterns.words.device)
    sch = aligner.scheme.struct()
    p, t = patterns.struct(), texts.struct()
    check(lib().nvb_banded_gotoh_score_best2(C.c_int(band_len), C.c_int(aligner.type), C.byref(sch), C.byref(p),
                                             C.c_void_p(quals.data_ptr()) if quals is not None else None, C.byref(t), C.c_uint32(n),
                                             C.c_uint32(distinct_dist), C.c_void_p(out.data_ptr()), _stream()), "nvb_banded_gotoh_score_best2")
    return out
