"""Seed + extend composition (examples/fmmap/fmmap.cu:255-400 shaped) over the C ABI."""
import ctypes as C
import ctypes.util
from dataclasses import dataclass, field
from typing import Optional
import torch
import numpy as np
from ._lib import (lib, check, SeedExtendParamsStruct, BestAlignmentOutStruct, PairParamsStruct, PairOutStruct, MapqParamsStruct, MapqOutStruct,
                   PairMapqOutStruct, AllParamsStruct, AllOutStruct, ReseedParamsStruct, ReseedOutStruct)
from .strings import PackedStringSet
from .fmindex import FMIndexDevice
from . import aln


@dataclass
class SeedExtendParams:
    seed_len: int = 20
    seed_interval: int = 10          # int(1 + 0.75*sqrtf(150)): nvBowtie's SimpleFunc evaluated on the host (params.cpp:157-158)
    band_len: int = 31
    type: int = aln.LOCAL
    both_strands: bool = True
    max_seed_hits: int = 100         # nvBowtie max_hits
    dedup_jobs: bool = True          # score identical (strand, window) jobs of a read once
    scheme: object = field(default_factory=lambda: aln.SimpleGotohScheme(2, -2, -5, -3))
    read_quals: Optional[torch.Tensor] = None   # uint8 base qualities indexed like the read symbols (with a QualityGotohScheme)

    def struct(self) -> SeedExtendParamsStruct:
        p = SeedExtendParamsStruct()
        p.seed_len, p.seed_interval, p.band_len, p.type = self.seed_len, self.seed_interval, self.band_len, self.type
        p.both_strands = 1 if self.both_strands else 0
        p.max_seed_hits = self.max_seed_hits
        p.dedup_jobs = 1 if self.dedup_jobs else 0
        p.scheme = self.scheme.struct()
        p.d_read_quals = self.read_quals.data_ptr() if self.read_quals is not None else None
        return p


_libm = None


def simple_func(kind: str, const: float, coeff: float, x) -> np.ndarray:
    """nvBowtie's SimpleFunc (nvBowtie/bowtie2/cuda/func.h:39-51), int32(const + coeff * f(float32(x))) with f = x ('L'), logf ('G') or
    sqrtf ('S'), in float32 like the reference's host code.  logf / sqrtf are the C library's (numpy's float32 log is a vectorised
    implementation picked by CPU features, so it is not guaranteed to round as the C library does).  Results outside the int32 range
    (x = 0 under 'G' gives -inf) are clamped to +-(2**31 - 1): INT_MIN stays the score of a read without an alignment."""
    global _libm
    if kind not in ("L", "G", "S"):
        raise ValueError("SimpleFunc type must be 'L', 'G' or 'S', not %r" % (kind,))
    if kind != "L" and _libm is None:
        _libm = C.CDLL(ctypes.util.find_library("m"))
        for f in (_libm.logf, _libm.sqrtf):
            f.restype, f.argtypes = C.c_float, [C.c_float]
    k, m = np.float32(const), np.float32(coeff)
    out = []
    for v in np.asarray(x, dtype=np.int64).reshape(-1):
        fx = np.float32(v)
        if kind == "G":
            fx = np.float32(_libm.logf(float(fx)))
        elif kind == "S":
            fx = np.float32(_libm.sqrtf(float(fx)))
        with np.errstate(invalid="ignore", over="ignore"):
            y = k + m * fx
        if np.isnan(y):
            raise ValueError("SimpleFunc %s,%g,%g is not a number at x = %d" % (kind, const, coeff, v))
        out.append(int(max(min(float(y), 2.0 ** 31 - 1), -(2.0 ** 31 - 1))))       # C truncation toward zero
    return np.array(out, dtype=np.int32)


@dataclass
class MapqParams:
    """Inputs of the second-best / MAPQ stage (nvb_mapq_params).  min_score: int32 tensor [max_read_len + 1] on the device, the minimum
    valid score of a read of each length (--score-min evaluated on the host); match_bonus: perfect_score(len) = len * match_bonus,
    0 = an end-to-end scheme (BowtieMapq2's monotone branch)."""
    min_score: torch.Tensor
    match_bonus: int

    @property
    def max_read_len(self) -> int:
        return self.min_score.numel() - 1

    @classmethod
    def from_score_min(cls, kind: str, const: float, coeff: float, max_read_len: int, match_bonus: int, device="cuda") -> "MapqParams":
        """nvBowtie's --score-min kind,const,coeff (kind 'L' linear, 'G' natural log, 'S' square root) for lengths 0 .. max_read_len"""
        tab = simple_func(kind, const, coeff, np.arange(max_read_len + 1))
        return cls(torch.from_numpy(tab).to(device), int(match_bonus))

    @classmethod
    def local(cls, max_read_len: int, device="cuda") -> "MapqParams":
        """nvBowtie's --local scheme: match bonus 2, --score-min G,0,10 (scoring_inl.h:81-99)"""
        return cls.from_score_min("G", 0.0, 10.0, max_read_len, 2, device)

    @classmethod
    def end_to_end(cls, max_read_len: int, device="cuda") -> "MapqParams":
        """nvBowtie's end-to-end scheme: no match bonus, --score-min L,-0.6,-0.6 (scoring_inl.h:107-122)"""
        return cls.from_score_min("L", -0.6, -0.6, max_read_len, 0, device)

    def struct(self) -> MapqParamsStruct:
        assert self.min_score.dtype == torch.int32 and self.min_score.is_cuda and self.min_score.is_contiguous()
        p = MapqParamsStruct()
        p.d_min_score, p.max_read_len, p.match_bonus = self.min_score.data_ptr(), self.max_read_len, self.match_bonus
        return p


class SeedExtendWorkspace:
    """pre-allocated outputs + temp storage for repeated calls on equally-shaped batches"""

    def __init__(self, fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams,
                 hit_capacity: int, keep_hits: bool = False, traceback: bool = False, mapq: Optional[MapqParams] = None):
        dev = fmi.device
        n = reads.count
        self.best_score = torch.empty(n, dtype=torch.int32, device=dev)
        self.best_pos = torch.empty(n, dtype=torch.int32, device=dev)
        self.n_hits = torch.zeros(3, dtype=torch.int32, device=dev)      # kept, found, distinct alignment jobs
        self.hit_capacity = hit_capacity
        self.hit_read = self.hit_window = self.hit_score = self.hit_sink = None
        if keep_hits:
            self.hit_read = torch.empty(hit_capacity, dtype=torch.int32, device=dev)
            self.hit_window = torch.empty((hit_capacity, 2), dtype=torch.int32, device=dev)
            self.hit_score = torch.empty(hit_capacity, dtype=torch.int32, device=dev)
            self.hit_sink = torch.empty((hit_capacity, 2), dtype=torch.int32, device=dev)
        # optional alignment (CIGAR ops, begin, strand) of every read's best hit
        self.best_ops = self.best_n_ops = self.best_begin = self.best_strand = None
        # an alignment's ops: one per read row (M or I) plus one per D, and M + D <= the window's length + band - 1 columns
        self.max_ops = 2 * reads.length + params.band_len
        if traceback:
            self.best_ops = torch.zeros((n, self.max_ops), dtype=torch.uint8, device=dev)
            self.best_n_ops = torch.zeros(n, dtype=torch.int32, device=dev)
            self.best_begin = torch.empty((n, 2), dtype=torch.int32, device=dev)
            self.best_strand = torch.empty(n, dtype=torch.uint8, device=dev)
        # optional second-best distinct alignment and MAPQ of every read
        self.mapq_params = mapq
        self.second_score = self.second_pos = self.second_strand = self.mapq = None
        if mapq is not None:
            self.second_score = torch.empty(n, dtype=torch.int32, device=dev)
            self.second_pos = torch.empty(n, dtype=torch.int32, device=dev)
            self.second_strand = torch.empty(n, dtype=torch.uint8, device=dev)
            self.mapq = torch.empty(n, dtype=torch.uint8, device=dev)
        tb = C.c_size_t(0)
        r = self._call(fmi, genome, reads, params, None, tb)
        if r != -2:
            check(r, "nvb_seed_extend(size query)")
        self.temp = torch.empty(tb.value, dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def _call(self, fmi, genome, reads, params, temp, tb):
        return _call(fmi, genome, reads, params, self, temp, tb)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _call(fmi, genome, reads, params, ws, temp, tb):
    s, rd, ps = fmi.struct(), reads.struct(), params.struct()
    ba = None
    if ws.best_ops is not None:
        ba = BestAlignmentOutStruct()
        ba.d_ops, ba.max_ops, ba.d_n_ops = ws.best_ops.data_ptr(), ws.max_ops, ws.best_n_ops.data_ptr()
        ba.d_begin, ba.d_strand = ws.best_begin.data_ptr(), ws.best_strand.data_ptr()
    if ws.mapq is not None:
        mp = ws.mapq_params.struct()
        mo = MapqOutStruct()
        mo.d_second_score, mo.d_second_pos = ws.second_score.data_ptr(), ws.second_pos.data_ptr()
        mo.d_second_strand, mo.d_mapq = ws.second_strand.data_ptr(), ws.mapq.data_ptr()
        return lib().nvb_seed_extend_mapq(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(reads.count), C.byref(ps),
                                          C.c_uint32(ws.hit_capacity), _p(ws.best_score), _p(ws.best_pos), _p(ws.n_hits),
                                          _p(ws.hit_read), _p(ws.hit_window), _p(ws.hit_score), _p(ws.hit_sink),
                                          C.byref(ba) if ba is not None else None, C.byref(mp), C.byref(mo),
                                          _p(temp), C.byref(tb), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    if ba is not None:
        return lib().nvb_seed_extend_traceback(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(reads.count), C.byref(ps),
                                               C.c_uint32(ws.hit_capacity), _p(ws.best_score), _p(ws.best_pos), _p(ws.n_hits),
                                               _p(ws.hit_read), _p(ws.hit_window), _p(ws.hit_score), _p(ws.hit_sink), C.byref(ba),
                                               _p(temp), C.byref(tb), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return lib().nvb_seed_extend(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(reads.count), C.byref(ps),
                                 C.c_uint32(ws.hit_capacity), _p(ws.best_score), _p(ws.best_pos), _p(ws.n_hits),
                                 _p(ws.hit_read), _p(ws.hit_window), _p(ws.hit_score), _p(ws.hit_sink),
                                 _p(temp), C.byref(tb), C.c_void_p(torch.cuda.current_stream().cuda_stream))


def seed_extend(fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams,
                workspace: Optional[SeedExtendWorkspace] = None, hit_capacity: Optional[int] = None, keep_hits: bool = False,
                traceback: bool = False, mapq: Optional[MapqParams] = None):
    """returns the workspace: .best_score[n], .best_pos[n], .n_hits[3] = (kept, total, distinct jobs), optional per-hit
    arrays, with traceback=True the alignment of every read's best hit (.best_ops END->START, .best_n_ops,
    .best_begin = (genome start, read start), .best_strand), and with mapq=MapqParams(...) the second-best distinct alignment and
    the mapping quality of every read (.second_score, .second_pos, .second_strand, .mapq; nvb_seed_extend_mapq).  A workspace made
    with mapq keeps computing them; a new mapq replaces its table for this and later calls"""
    if workspace is None:
        if hit_capacity is None:
            hit_capacity = 32 * reads.count + 1024
        workspace = SeedExtendWorkspace(fmi, genome, reads, params, hit_capacity, keep_hits, traceback, mapq)
    elif mapq is not None:
        if workspace.mapq is None:
            raise ValueError("seed_extend(mapq=...): the workspace was created without mapq outputs")
        workspace.mapq_params = mapq
    tb = C.c_size_t(workspace.temp_bytes)
    check(_call(fmi, genome, reads, params, workspace, workspace.temp, tb), "nvb_seed_extend")
    return workspace


@dataclass
class ReseedParams:
    """Reseeding rounds of seed_extend_reseed (nvb_reseed_params): max_reseed rounds after the first (nvBowtie -R), rep_seeds (nvBowtie
    --rep-seeds) and min_score, an int32 tensor [max_read_len + 1] on the device: a read counts as aligned when its best score reaches
    min_score[len] (--score-min evaluated on the host, as MapqParams.min_score)."""
    min_score: torch.Tensor
    max_reseed: int = 2
    rep_seeds: int = 300

    @property
    def max_read_len(self) -> int:
        return self.min_score.numel() - 1

    @classmethod
    def from_score_min(cls, kind: str, const: float, coeff: float, max_read_len: int, max_reseed: int = 2, rep_seeds: int = 300,
                       device="cuda") -> "ReseedParams":
        """nvBowtie's --score-min kind,const,coeff for lengths 0 .. max_read_len (see MapqParams.from_score_min)"""
        tab = simple_func(kind, const, coeff, np.arange(max_read_len + 1))
        return cls(torch.from_numpy(tab).to(device), int(max_reseed), int(rep_seeds))

    @classmethod
    def local(cls, max_read_len: int, max_reseed: int = 2, rep_seeds: int = 300, device="cuda") -> "ReseedParams":
        """nvBowtie's --local min score, G,0,10"""
        return cls.from_score_min("G", 0.0, 10.0, max_read_len, max_reseed, rep_seeds, device)

    @classmethod
    def end_to_end(cls, max_read_len: int, max_reseed: int = 2, rep_seeds: int = 300, device="cuda") -> "ReseedParams":
        """nvBowtie's end-to-end min score, L,-0.6,-0.6"""
        return cls.from_score_min("L", -0.6, -0.6, max_read_len, max_reseed, rep_seeds, device)

    def struct(self) -> ReseedParamsStruct:
        assert self.min_score.dtype == torch.int32 and self.min_score.is_cuda and self.min_score.is_contiguous()
        p = ReseedParamsStruct()
        p.max_reseed, p.rep_seeds, p.d_min_score, p.max_read_len = self.max_reseed, self.rep_seeds, self.min_score.data_ptr(), self.max_read_len
        return p


class ReseedWorkspace(SeedExtendWorkspace):
    """SeedExtendWorkspace of seed_extend_reseed: the same fields, plus .rounds[n] (the rounds each read was seeded in) and
    .active[max_reseed + 1] (the reads seeded in each round)"""

    def __init__(self, fmi, genome, reads, params, hit_capacity, reseed: ReseedParams, keep_hits=False, traceback=False, mapq=None):
        self.reseed = reseed
        self.rounds = torch.empty(max(reads.count, 1), dtype=torch.uint8, device=fmi.device)[:reads.count]
        self.active = torch.zeros(reseed.max_reseed + 1, dtype=torch.int32, device=fmi.device)
        super().__init__(fmi, genome, reads, params, hit_capacity, keep_hits, traceback, mapq)

    def _call(self, fmi, genome, reads, params, temp, tb):
        s, rd, ps, rp = fmi.struct(), reads.struct(), params.struct(), self.reseed.struct()
        ro = ReseedOutStruct()
        ro.d_rounds, ro.d_active = _storage_ptr(self.rounds), self.active.data_ptr()
        ba = mp = mo = None
        if self.best_ops is not None:
            ba = BestAlignmentOutStruct()
            ba.d_ops, ba.max_ops, ba.d_n_ops = self.best_ops.data_ptr(), self.max_ops, self.best_n_ops.data_ptr()
            ba.d_begin, ba.d_strand = self.best_begin.data_ptr(), self.best_strand.data_ptr()
        if self.mapq is not None:
            mp = self.mapq_params.struct()
            mo = MapqOutStruct()
            mo.d_second_score, mo.d_second_pos = self.second_score.data_ptr(), self.second_pos.data_ptr()
            mo.d_second_strand, mo.d_mapq = self.second_strand.data_ptr(), self.mapq.data_ptr()
        ref = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return lib().nvb_seed_extend_reseed(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(reads.count), C.byref(ps),
                                            C.c_uint32(self.hit_capacity), _p(self.best_score), _p(self.best_pos), _p(self.n_hits),
                                            _p(self.hit_read), _p(self.hit_window), _p(self.hit_score), _p(self.hit_sink),
                                            ref(ba), ref(mp), ref(mo), C.byref(rp), C.byref(ro),
                                            _p(temp), C.byref(tb), C.c_void_p(torch.cuda.current_stream().cuda_stream))


def seed_extend_reseed(fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams, reseed: ReseedParams,
                       traceback: bool = False, mapq: Optional[MapqParams] = None, keep_hits: bool = False,
                       workspace: Optional[ReseedWorkspace] = None, hit_capacity: Optional[int] = None) -> ReseedWorkspace:
    """seed_extend with nvBowtie's reseeding rounds (nvb_seed_extend_reseed): reads whose seeds found nothing, only repeats, or no
    alignment reaching reseed.min_score are seeded again at shifted offsets, up to reseed.max_reseed more times, and every round's
    alignments compete for each read's best, second best and MAPQ.  Returns a ReseedWorkspace: seed_extend's fields plus .rounds and
    .active.  The call synchronises the stream once per round after the first.  A workspace of an equally-shaped earlier call is reused
    (reseed and mapq replace its parameters)"""
    if workspace is None:
        if hit_capacity is None:
            hit_capacity = 32 * reads.count + 1024
        workspace = ReseedWorkspace(fmi, genome, reads, params, hit_capacity, reseed, keep_hits, traceback, mapq)
    else:
        if reseed.max_reseed + 1 > workspace.active.numel():
            raise ValueError("seed_extend_reseed: the workspace was created for at most %d rounds" % workspace.active.numel())
        workspace.reseed = reseed
        if mapq is not None:
            if workspace.mapq is None:
                raise ValueError("seed_extend_reseed(mapq=...): the workspace was created without mapq outputs")
            workspace.mapq_params = mapq
    tb = C.c_size_t(workspace.temp_bytes)
    check(workspace._call(fmi, genome, reads, params, workspace.temp, tb), "nvb_seed_extend_reseed")
    return workspace


def _storage_ptr(t):
    """the address of t's first element, also for an empty view of a non-empty allocation (whose data_ptr() is 0)"""
    return t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


class AllAlignments:
    """Up to max_per_read distinct alignments of every read (nvb_seed_extend_all), each traced.  Per read (n): .best_score, .best_pos,
    .second_score, .second_pos, .second_strand, .mapq (those of seed_extend(mapq=...)), .first[n + 1] (read r's alignments are
    [first[r], first[r + 1])) and .n_hits[3]; per alignment slot (capacity): .read, .score, .pos (end), .ops[., max_ops] (END->START),
    .n_ops, .begin = (genome start, read start), .strand; .count = (stored, wanted).  Only the first count[0] slots are written."""

    def __init__(self, fmi, genome, reads: PackedStringSet, params: SeedExtendParams, mapq: MapqParams, max_per_read: int, capacity: int,
                 hit_capacity: int):
        dev = fmi.device
        n = reads.count
        self.n_reads, self.max_per_read, self.capacity, self.hit_capacity = n, int(max_per_read), int(capacity), int(hit_capacity)
        self.mapq_params = mapq
        per_read = lambda dt: torch.empty(max(n, 1), dtype=dt, device=dev)[:n]     # noqa: E731  (never a NULL pointer)
        self.best_score, self.best_pos = per_read(torch.int32), per_read(torch.int32)
        self.n_hits = torch.zeros(3, dtype=torch.int32, device=dev)
        self.second_score, self.second_pos = per_read(torch.int32), per_read(torch.int32)
        self.second_strand, self.mapq = per_read(torch.uint8), per_read(torch.uint8)
        self.max_ops = 2 * reads.length + params.band_len             # (as SeedExtendWorkspace)
        c = self.capacity
        self.first = torch.empty(n + 1, dtype=torch.int32, device=dev)
        self.read = torch.empty(c, dtype=torch.int32, device=dev)
        self.score = torch.empty(c, dtype=torch.int32, device=dev)
        self.pos = torch.empty(c, dtype=torch.int32, device=dev)
        self.ops = torch.zeros((c, self.max_ops), dtype=torch.uint8, device=dev)
        self.n_ops = torch.zeros(c, dtype=torch.int32, device=dev)
        self.begin = torch.empty((c, 2), dtype=torch.int32, device=dev)
        self.strand = torch.empty(c, dtype=torch.uint8, device=dev)
        self.count = torch.zeros(2, dtype=torch.int32, device=dev)
        tb = C.c_size_t(0)
        r = self._call(fmi, genome, reads, params, None, tb)
        if r != -2:
            check(r, "nvb_seed_extend_all(size query)")
        self.temp = torch.empty(tb.value, dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def _call(self, fmi, genome, reads, params, temp, tb):
        s, rd, ps, mp = fmi.struct(), reads.struct(), params.struct(), self.mapq_params.struct()
        mo = MapqOutStruct()
        mo.d_second_score, mo.d_second_pos = _storage_ptr(self.second_score), _storage_ptr(self.second_pos)
        mo.d_second_strand, mo.d_mapq = _storage_ptr(self.second_strand), _storage_ptr(self.mapq)
        ap = AllParamsStruct()
        ap.max_per_read, ap.capacity = self.max_per_read, self.capacity
        ao = AllOutStruct()
        ao.d_first, ao.d_read, ao.d_score, ao.d_pos = self.first.data_ptr(), self.read.data_ptr(), self.score.data_ptr(), self.pos.data_ptr()
        ao.alignment.d_ops, ao.alignment.max_ops, ao.alignment.d_n_ops = self.ops.data_ptr(), self.max_ops, self.n_ops.data_ptr()
        ao.alignment.d_begin, ao.alignment.d_strand = self.begin.data_ptr(), self.strand.data_ptr()
        ao.d_count = self.count.data_ptr()
        return lib().nvb_seed_extend_all(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(reads.count), C.byref(ps), C.c_uint32(self.hit_capacity),
                                         C.c_void_p(_storage_ptr(self.best_score)), C.c_void_p(_storage_ptr(self.best_pos)), _p(self.n_hits),
                                         None, None, None, None, None,
                                         C.byref(mp), C.byref(mo), C.byref(ap), C.byref(ao), _p(temp), C.byref(tb),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))

    def run(self, fmi, genome, reads, params):
        tb = C.c_size_t(self.temp_bytes)
        check(self._call(fmi, genome, reads, params, self.temp, tb), "nvb_seed_extend_all")
        return self

    def strings(self, reads: PackedStringSet) -> PackedStringSet:
        """the reads of the capacity alignment slots as a string set over the reads' own words (string i = read read[i]; slots past
        count[0] point at read 0): the `reads` of finish_alignments over these alignments"""
        n = reads.count
        idx = self.read.long().clamp(0, max(n - 1, 0))
        if int(self.count[0]) < self.capacity:
            idx = torch.where(torch.arange(self.capacity, device=idx.device) < self.count[0], idx, torch.zeros_like(idx))
        if reads.offsets is not None:
            offsets = reads.offsets[idx] if n else torch.zeros(self.capacity, dtype=torch.int32, device=idx.device)
        else:
            offsets = (idx * reads.stride).to(torch.int32)
        lengths = reads.lengths[idx] if reads.lengths is not None and n else torch.full((self.capacity,), reads.length, dtype=torch.int32,
                                                                                          device=idx.device)
        return PackedStringSet(words=reads.words, bits=reads.bits, big_endian=reads.big_endian, offsets=offsets.contiguous(),
                               lengths=lengths.contiguous(), stride=0, length=reads.length, count=self.capacity)


    def bam_records(self, genome: torch.Tensor, genome_len: int, reads: PackedStringSet, contigs, names, quals: Optional[torch.Tensor] = None,
                    capacity: Optional[int] = None):
        """finish_alignments over the alignment slots, then their BAM records (bam_records_all: primary, secondary and unmapped records,
        NH); the returned BamRecords is what write_sorted_bam / bgzf_compress take"""
        from .finish import finish_alignments
        from .bam import bam_records_all
        f = finish_alignments(genome, self.strings(reads), self.ops, self.n_ops, self.begin, self.strand, genome_len=genome_len)
        return bam_records_all(self, f, reads, contigs, names, quals=quals, capacity=capacity)


def seed_extend_all(fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams, mapq: MapqParams,
                    max_per_read: int, capacity: Optional[int] = None, hit_capacity: Optional[int] = None,
                    workspace: Optional[AllAlignments] = None) -> AllAlignments:
    """up to max_per_read distinct alignments of every read (0 = every distinct alignment: nvBowtie's --all), traced, with the
    best / second-best / MAPQ outputs of seed_extend(mapq=...).  capacity: alignment slots, by default max_per_read * n_reads + 1024
    (16 per read for max_per_read = 0), at most hit_capacity; .count[1] > .count[0] tells that reads were left out.  The call traces in
    ceil(capacity / n_reads) slices of n_reads, each a few kernel launches even when empty, so a capacity far above the alignments
    expected costs launches.  A workspace of an equally-shaped earlier call is reused as it is"""
    if workspace is None:
        if hit_capacity is None:
            hit_capacity = 32 * reads.count + 1024
        if capacity is None:
            capacity = min((int(max_per_read) or 16) * reads.count + 1024, hit_capacity)
        workspace = AllAlignments(fmi, genome, reads, params, mapq, max_per_read, capacity, hit_capacity)
    return workspace.run(fmi, genome, reads, params)


PAIR_UNPAIRED, PAIR_CONCORDANT, PAIR_RESCUED_MATE1, PAIR_RESCUED_MATE2, PAIR_DISCORDANT = 0, 1, 2, 4, 8
# nvb_pair_params.policy (NVB_PE_*) and flags
PE_POLICIES = ("fr", "rf", "ff", "rr")
PE_NO_OVERLAP, PE_DISCORDANT, PE_NO_MIXED = 1, 2, 4


@dataclass
class PairParams:
    """fragment constraints and pairing options of the paired-end stage (nvBowtie --minins / --maxins, --fr / --rf / --ff / --rr,
    --no-overlap, --no-mixed and discordant pairs; include/nvbio_b200.h nvb_pair_params).  policy: the mates' orientation; overlap=False:
    a concordant pair's mates may not overlap and the rescue looks only past the anchor; discordant=True (needs mapq): an unpaired pair
    whose two mates align uniquely is reported as PAIR_DISCORDANT; mixed=False: the mates of a pair that is still unpaired are reported
    unaligned.  The defaults are the FR pairing with overlap, no discordant pairs and unpaired mates reported."""
    min_frag: int = 0
    max_frag: int = 500
    min_mate_score: int = 60          # a mate's alignment (anchor or rescued) must reach this score to take part in a pair
    rescue_capacity: Optional[int] = None
    policy: str = "fr"
    overlap: bool = True
    discordant: bool = False
    mixed: bool = True

    @property
    def policy_code(self) -> int:
        """NVB_PE_FR 0, NVB_PE_RF 1, NVB_PE_FF 2, NVB_PE_RR 3"""
        if self.policy not in PE_POLICIES:
            raise ValueError("PairParams.policy must be one of %s, not %r" % (PE_POLICIES, self.policy))
        return PE_POLICIES.index(self.policy)

    @property
    def flags(self) -> int:
        return (0 if self.overlap else PE_NO_OVERLAP) | (PE_DISCORDANT if self.discordant else 0) | (0 if self.mixed else PE_NO_MIXED)

    def struct(self, n_pairs) -> PairParamsStruct:
        p = PairParamsStruct()
        p.min_frag, p.max_frag, p.min_mate_score = self.min_frag, self.max_frag, self.min_mate_score
        p.rescue_capacity = 2 * n_pairs if self.rescue_capacity is None else self.rescue_capacity
        p.policy, p.flags = self.policy_code, self.flags
        return p


class PairedWorkspace:
    """outputs + temp storage of seed_extend_paired for repeated calls on equally-shaped batches"""

    def __init__(self, fmi, genome, reads: PackedStringSet, params: SeedExtendParams, pair: PairParams, hit_capacity: int,
                 mapq: Optional[MapqParams] = None, traceback: bool = False, max_ops: Optional[int] = None):
        dev = fmi.device
        assert reads.count % 2 == 0
        self.n_pairs = n = reads.count // 2
        self.hit_capacity = hit_capacity
        self.pair_score = torch.empty(n, dtype=torch.int32, device=dev)
        self.pair_flags = torch.empty(n, dtype=torch.int32, device=dev)
        self.mate_score = torch.empty((2, n), dtype=torch.int32, device=dev)
        self.mate_pos = torch.empty((2, n), dtype=torch.int32, device=dev)
        self.mate_strand = torch.empty((2, n), dtype=torch.uint8, device=dev)
        self.n_rescue = torch.zeros(2, dtype=torch.int32, device=dev)
        self.n_hits = torch.zeros(3, dtype=torch.int32, device=dev)
        # optional second-best pair and MAPQ of every mate
        self.mapq_params = mapq
        self.second_pair_score = self.second_mate_pos = self.second_mate_strand = self.mate_second_score = self.mate_mapq = None
        if mapq is not None:
            self.second_pair_score = torch.empty(n, dtype=torch.int32, device=dev)
            self.second_mate_pos = torch.empty((2, n), dtype=torch.int32, device=dev)
            self.second_mate_strand = torch.empty((2, n), dtype=torch.uint8, device=dev)
            self.mate_second_score = torch.empty((2, n), dtype=torch.int32, device=dev)
            self.mate_mapq = torch.empty((2, n), dtype=torch.uint8, device=dev)
        # optional alignment of both mates (nvb_seed_extend_paired_traceback)
        self.mate_ops = self.mate_n_ops = self.mate_begin = None
        self.max_ops = 2 * reads.length + params.band_len if max_ops is None else max_ops      # (as SeedExtendWorkspace)
        if traceback:
            self.mate_ops = torch.zeros((2, n, self.max_ops), dtype=torch.uint8, device=dev)
            self.mate_n_ops = torch.zeros((2, n), dtype=torch.int32, device=dev)
            self.mate_begin = torch.empty((2, n, 2), dtype=torch.int32, device=dev)
        tb = C.c_size_t(0)
        r = self._call(fmi, genome, reads, params, pair, None, tb)
        if r != -2:
            check(r, "nvb_seed_extend_paired(size query)")
        self.temp = torch.empty(tb.value, dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def _call(self, fmi, genome, reads, params, pair, temp, tb):
        return _call_paired(fmi, genome, reads, params, pair, self, temp, tb)


def _call_paired(fmi, genome, reads, params, pair, ws, temp, tb, reseed=None):
    s, rd, ps, pp = fmi.struct(), reads.struct(), params.struct(), pair.struct(ws.n_pairs)
    po = PairOutStruct()
    po.d_pair_score, po.d_pair_flags = ws.pair_score.data_ptr(), ws.pair_flags.data_ptr()
    po.d_mate_score, po.d_mate_pos, po.d_mate_strand = ws.mate_score.data_ptr(), ws.mate_pos.data_ptr(), ws.mate_strand.data_ptr()
    po.d_n_rescue = ws.n_rescue.data_ptr()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    mp = mo = None
    if ws.mate_mapq is not None:
        mp = ws.mapq_params.struct()
        mo = PairMapqOutStruct()
        mo.d_second_pair_score, mo.d_second_mate_pos = ws.second_pair_score.data_ptr(), ws.second_mate_pos.data_ptr()
        mo.d_second_mate_strand, mo.d_mate_second_score = ws.second_mate_strand.data_ptr(), ws.mate_second_score.data_ptr()
        mo.d_mate_mapq = ws.mate_mapq.data_ptr()
    ba = None
    if ws.mate_ops is not None:
        ba = BestAlignmentOutStruct()
        ba.d_ops, ba.max_ops, ba.d_n_ops = ws.mate_ops.data_ptr(), ws.max_ops, ws.mate_n_ops.data_ptr()
        ba.d_begin, ba.d_strand = ws.mate_begin.data_ptr(), None
    if reseed is not None:
        rp, ro = reseed.struct(), ReseedOutStruct()
        ro.d_rounds, ro.d_active = _storage_ptr(ws.rounds), ws.active.data_ptr()
        ref = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return lib().nvb_seed_extend_paired_reseed(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(ws.n_pairs), C.byref(ps),
                                                   C.c_uint32(ws.hit_capacity), C.byref(pp), C.byref(po), ref(ba), ref(mp), ref(mo),
                                                   C.byref(rp), C.byref(ro), _p(ws.n_hits), _p(temp), C.byref(tb), stream)
    if ba is not None:
        return lib().nvb_seed_extend_paired_traceback(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(ws.n_pairs), C.byref(ps),
                                                      C.c_uint32(ws.hit_capacity), C.byref(pp), C.byref(po), C.byref(ba),
                                                      C.byref(mp) if mp is not None else None, C.byref(mo) if mo is not None else None,
                                                      _p(ws.n_hits), _p(temp), C.byref(tb), stream)
    if mo is not None:
        return lib().nvb_seed_extend_paired_mapq(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(ws.n_pairs), C.byref(ps),
                                                 C.c_uint32(ws.hit_capacity), C.byref(pp), C.byref(po), C.byref(mp), C.byref(mo),
                                                 _p(ws.n_hits), _p(temp), C.byref(tb), stream)
    return lib().nvb_seed_extend_paired(C.byref(s), _p(genome), C.byref(rd), C.c_uint32(ws.n_pairs), C.byref(ps), C.c_uint32(ws.hit_capacity),
                                        C.byref(pp), C.byref(po), _p(ws.n_hits), _p(temp), C.byref(tb), stream)


def seed_extend_paired(fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams, pair: PairParams,
                       workspace: Optional[PairedWorkspace] = None, hit_capacity: Optional[int] = None, mapq: Optional[MapqParams] = None,
                       traceback: bool = False):
    """paired-end seed + extend (reads = mate 1 of every pair, then mate 2 of every pair): concordant pairs straight from the two
    independent alignments, opposite-mate full-DP rescue for the rest (nvBowtie's best-approx paired flow,
    score_opposite_inl.h:90-266).  Returns the workspace: .pair_score[n], .pair_flags[n], .mate_score/.mate_pos/.mate_strand[2,n],
    .n_rescue[2] = (full-DP jobs run, wanted).  With mapq=MapqParams(...) also the second-best pair and the MAPQ of every mate
    (nvb_seed_extend_paired_mapq): .second_pair_score[n], .second_mate_pos/.second_mate_strand[2,n], .mate_second_score[2,n] (each mate's
    single-end second score) and .mate_mapq[2,n].  A workspace made with mapq keeps computing them; a new mapq replaces its table.
    With traceback=True also the alignment of every mate (nvb_seed_extend_paired_traceback): .mate_ops[2,n,max_ops] (END->START, 0 M,
    1 I, 2 D), .mate_n_ops[2,n] and .mate_begin[2,n,2] = (genome start, read start) -- a rescued mate's from the full-matrix DP that
    placed it.  A workspace made with traceback keeps computing them"""
    if workspace is None:
        if hit_capacity is None:
            hit_capacity = 32 * reads.count + 1024
        workspace = PairedWorkspace(fmi, genome, reads, params, pair, hit_capacity, mapq, traceback)
    elif traceback and workspace.mate_ops is None:
        raise ValueError("seed_extend_paired(traceback=True): the workspace was created without traceback outputs")
    elif mapq is not None:
        if workspace.mate_mapq is None:
            raise ValueError("seed_extend_paired(mapq=...): the workspace was created without mapq outputs")
        workspace.mapq_params = mapq
    tb = C.c_size_t(workspace.temp_bytes)
    check(_call_paired(fmi, genome, reads, params, pair, workspace, workspace.temp, tb), "nvb_seed_extend_paired")
    return workspace


class PairedReseedWorkspace(PairedWorkspace):
    """PairedWorkspace of seed_extend_paired_reseed: the same fields, plus .rounds[2, n] (the rounds each mate was seeded in) and
    .active[max_reseed + 1] (the mates seeded in each round)"""

    def __init__(self, fmi, genome, reads, params, pair, hit_capacity, reseed: ReseedParams, mapq=None, traceback=False):
        self.reseed = reseed
        n = reads.count // 2
        self.rounds = torch.empty(max(2 * n, 1), dtype=torch.uint8, device=fmi.device)[:2 * n].view(2, n)
        self.active = torch.zeros(reseed.max_reseed + 1, dtype=torch.int32, device=fmi.device)
        super().__init__(fmi, genome, reads, params, pair, hit_capacity, mapq, traceback)

    def _call(self, fmi, genome, reads, params, pair, temp, tb):
        return _call_paired(fmi, genome, reads, params, pair, self, temp, tb, reseed=self.reseed)


def seed_extend_paired_reseed(fmi: FMIndexDevice, genome: torch.Tensor, reads: PackedStringSet, params: SeedExtendParams, pair: PairParams,
                              reseed: ReseedParams, mapq: Optional[MapqParams] = None, traceback: bool = False,
                              workspace: Optional[PairedReseedWorkspace] = None, hit_capacity: Optional[int] = None) -> PairedReseedWorkspace:
    """seed_extend_paired with nvBowtie's reseeding rounds (nvb_seed_extend_paired_reseed): mates whose seeds found nothing or only
    repeats are seeded again at shifted offsets, up to reseed.max_reseed more times (reseed.min_score is not read: the paired flags are
    the seed statistics alone), and the pairing, rescue, paired MAPQ and mate tracebacks then run once over every round's alignments.
    Returns a PairedReseedWorkspace: seed_extend_paired's fields plus .rounds[2, n] and .active.  The call synchronises the stream once
    per round after the first.  A workspace of an equally-shaped earlier call is reused (reseed and mapq replace its parameters)"""
    if workspace is None:
        if hit_capacity is None:
            hit_capacity = 32 * reads.count + 1024
        workspace = PairedReseedWorkspace(fmi, genome, reads, params, pair, hit_capacity, reseed, mapq, traceback)
    else:
        if reseed.max_reseed + 1 > workspace.active.numel():
            raise ValueError("seed_extend_paired_reseed: the workspace was created for at most %d rounds" % workspace.active.numel())
        if traceback and workspace.mate_ops is None:
            raise ValueError("seed_extend_paired_reseed(traceback=True): the workspace was created without traceback outputs")
        workspace.reseed = reseed
        if mapq is not None:
            if workspace.mate_mapq is None:
                raise ValueError("seed_extend_paired_reseed(mapq=...): the workspace was created without mapq outputs")
            workspace.mapq_params = mapq
    tb = C.c_size_t(workspace.temp_bytes)
    check(workspace._call(fmi, genome, reads, params, pair, workspace.temp, tb), "nvb_seed_extend_paired_reseed")
    return workspace


STAGES = ("strings", "seed_match", "hit_slots", "locate_windows", "dedup", "extend", "reduce")


def last_stage_ms():
    """device time (ms) of the stages of the most recent seed_extend call"""
    ms = (C.c_float * 7)()
    check(lib().nvb_seed_extend_stage_ms(ms), "nvb_seed_extend_stage_ms")
    return dict(zip(STAGES, [float(v) for v in ms]))


def _host_view(ptr, count, dtype):
    """a torch tensor over `count` elements of pinned host memory owned by the C library (no copy)"""
    nbytes = count * torch.tensor([], dtype=dtype).element_size()
    buf = (C.c_char * nbytes).from_address(ptr)
    return torch.frombuffer(buf, dtype=dtype, count=count)


class StreamingSeedExtend:
    """Host-to-host batches through the C ABI's nvb_pipeline (include/nvbio_b200.h): the production entry point that replaces
    nvBowtie's input thread -> compute thread hand-off (nvBowtie/bowtie2/cuda/compute_thread.cu:213-243) and its per-stage
    cudaDeviceSynchronize.

    `submit(host_words)` enqueues H2D copy -> seed_extend[_paired] -> D2H copy of the per-read results and returns a ticket;
    `result(ticket)` waits for that batch only.  `depth` batches are in flight: copies overlap kernels, and consecutive batches
    run on different compute streams.  host_words: int32 tensor [n_reads, words_per_read] in host memory (pinned = async copy).
    pair: PairParams for paired-end batches (reads = mate 1 of every pair, then mate 2)."""

    def __init__(self, fmi: FMIndexDevice, genome: torch.Tensor, params: SeedExtendParams, n_reads: int, read_len: int,
                 words_per_read: int, hit_capacity: Optional[int] = None, depth: int = 2, bits: int = 2, pair: Optional["PairParams"] = None):
        self.fmi, self.genome, self.params, self.pair = fmi, genome, params, pair          # keep the device buffers alive
        self.n_reads, self.read_len, self.wpr, self.bits, self.depth = n_reads, read_len, words_per_read, bits, depth
        if hit_capacity is None:
            hit_capacity = 32 * n_reads + 1024
        self._params_struct = params.struct()
        s = fmi.struct()
        pp = pair.struct(n_reads // 2) if pair is not None else None
        self._h = C.c_void_p()
        with torch.cuda.device(fmi.device):
            check(lib().nvb_pipeline_create(C.byref(s), C.c_void_p(genome.data_ptr()), C.byref(self._params_struct),
                                            C.byref(pp) if pp is not None else None,
                                            C.c_uint32(n_reads), C.c_uint32(read_len), C.c_uint32(words_per_read), C.c_uint32(bits),
                                            C.c_uint32(hit_capacity), C.c_uint32(depth), C.byref(self._h)), "nvb_pipeline_create")
        h2d, d2h = C.c_size_t(0), C.c_size_t(0)
        lib().nvb_pipeline_traffic(self._h, C.byref(h2d), C.byref(d2h))
        self.h2d_bytes, self.d2h_bytes = int(h2d.value), int(d2h.value)
        self._keep = {}
        self.last_device_ms = None

    def submit(self, host_words: torch.Tensor) -> int:
        assert not host_words.is_cuda and host_words.is_contiguous() and host_words.numel() == self.n_reads * self.wpr
        t = C.c_uint32(0)
        check(lib().nvb_pipeline_submit(self._h, C.c_void_p(host_words.data_ptr()), C.byref(t)), "nvb_pipeline_submit")
        self._keep[int(t.value)] = host_words                # the copy is asynchronous: keep the source alive until result()
        return int(t.value)

    def result(self, ticket: int):
        """single end: (best_score[n], best_pos[n], n_hits[3]); paired: dict of the nvb_pair_out arrays -- views of the pipeline's
        pinned host buffers, valid until `depth` further batches have been submitted"""
        from ._lib import PipelineResultStruct
        r = PipelineResultStruct()
        check(lib().nvb_pipeline_wait(self._h, C.c_uint32(ticket), C.byref(r)), "nvb_pipeline_wait")
        self._keep.pop(ticket, None)
        self.last_device_ms = float(r.device_ms)
        n = self.n_reads
        if self.pair is None:
            return _host_view(r.best_score, n, torch.int32), _host_view(r.best_pos, n, torch.int32), _host_view(r.n_hits, 3, torch.int32)
        return dict(pair_score=_host_view(r.pair_score, n // 2, torch.int32), pair_flags=_host_view(r.pair_flags, n // 2, torch.int32),
                    mate_score=_host_view(r.mate_score, n, torch.int32).view(2, n // 2), mate_pos=_host_view(r.mate_pos, n, torch.int32).view(2, n // 2),
                    mate_strand=_host_view(r.mate_strand, n, torch.uint8).view(2, n // 2), n_rescue=_host_view(r.n_rescue, 2, torch.int32),
                    n_hits=_host_view(r.n_hits, 3, torch.int32))

    def close(self):
        if self._h:
            lib().nvb_pipeline_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class StreamingBam:
    """Host reads in, BAM out: the BAM mode of nvb_pipeline (nvb_pipeline_create_bam, include/nvbio_b200.h).  Every batch runs mapping with
    MAPQ and traceback (seed_extend(traceback=True, mapq=...) or seed_extend_paired(traceback=True, mapq=...)), finish_alignments,
    bam_records and, with compress=True, bgzf_compress on the device, `depth` batches in flight; only the batch's counts and its payload
    (exactly its byte count) come back.  The payload equals what that chain gives for the batch: the record stream, or its BGZF members,
    which write_bam writes verbatim.

    max_reads: reads per batch at most (paired: mates, mate 1 of every pair then mate 2); contigs: a ContigTable of the genome; mapq: the
    MapqParams of the mapping call (max_read_len >= read_len); pair: PairParams for paired batches (every policy and flag, discordant pairs
    included); quals / lengths: every submit passes base qualities / per-read lengths; max_name_bytes: bytes of names per batch (default 64
    per name); max_ops / max_cigar / max_md: 0 = never truncate (2 * read_len + band_len, max_ops + 2, 3 * max_ops + 1, the defaults of
    seed_extend / finish_alignments).  .slot_bytes is the device memory one slot holds."""

    def __init__(self, fmi: FMIndexDevice, genome: torch.Tensor, params: SeedExtendParams, max_reads: int, read_len: int, words_per_read: int,
                 contigs, mapq: MapqParams, pair: Optional[PairParams] = None, quals: bool = False, lengths: bool = False, compress: bool = True,
                 depth: int = 2, bits: int = 2, hit_capacity: Optional[int] = None, max_name_bytes: Optional[int] = None,
                 max_ops: int = 0, max_cigar: int = 0, max_md: int = 0):
        from ._lib import PipelineBamParamsStruct
        if params.read_quals is not None:
            raise ValueError("StreamingBam: qualities come with every batch (quals=True), not in params.read_quals")
        self.fmi, self.genome, self.params, self.pair, self.contigs, self.mapq = fmi, genome, params, pair, contigs, mapq   # keep alive
        self.max_reads, self.read_len, self.wpr, self.bits, self.depth = int(max_reads), int(read_len), int(words_per_read), int(bits), int(depth)
        self.quals, self.lengths, self.compress = bool(quals), bool(lengths), bool(compress)
        self.n_names = self.max_reads // 2 if pair is not None else self.max_reads
        self.max_name_bytes = int(max_name_bytes) if max_name_bytes is not None else 64 * max(self.n_names, 1)
        if hit_capacity is None:
            hit_capacity = 32 * self.max_reads + 1024
        self._params_struct = params.struct()
        self._mapq_struct = mapq.struct()
        self._contig_dev = contigs.device(fmi.device)
        bp = self._bam_struct = PipelineBamParamsStruct()
        bp.mapq = C.addressof(self._mapq_struct)
        bp.d_contig_begin, bp.n_contigs = self._contig_dev.data_ptr(), len(contigs.names)
        bp.max_name_bytes, bp.has_quals, bp.has_lengths, bp.compress = self.max_name_bytes, int(self.quals), int(self.lengths), int(self.compress)
        bp.max_ops, bp.max_cigar, bp.max_md = int(max_ops), int(max_cigar), int(max_md)
        s = fmi.struct()
        pp = pair.struct(self.max_reads // 2) if pair is not None else None
        self._h = C.c_void_p()
        with torch.cuda.device(fmi.device):
            check(lib().nvb_pipeline_create_bam(C.byref(s), C.c_void_p(genome.data_ptr()), C.byref(self._params_struct),
                                                C.byref(pp) if pp is not None else None, C.byref(bp),
                                                C.c_uint32(self.max_reads), C.c_uint32(self.read_len), C.c_uint32(self.wpr), C.c_uint32(self.bits),
                                                C.c_uint32(hit_capacity), C.c_uint32(self.depth), C.byref(self._h)), "nvb_pipeline_create_bam")
        self.slot_bytes = int(lib().nvb_pipeline_slot_bytes(self._h))
        self._keep = {}
        self.last_device_ms = None

    @staticmethod
    def _host(a, dtype, what):
        t = torch.as_tensor(a)
        if t.is_cuda:
            raise ValueError("StreamingBam.submit: %s must be in host memory" % what)
        t = t.contiguous()
        if t.dtype == dtype:
            return t
        if t.element_size() == torch.tensor([], dtype=dtype).element_size():
            return t.view(dtype)                                  # (uint32 words / lengths: the same bits)
        return t.to(dtype)

    def submit(self, words, names, quals=None, lengths=None, n: Optional[int] = None) -> int:
        """enqueue one batch and return its ticket.  words: int32 [n, words_per_read] in host memory (pinned = asynchronous copy); names:
        one per read (per pair when paired), str or bytes, or the (bytes, offsets) pair of bam.pack_names; quals: uint8 [n, symbols per
        read] (words_per_read * 32 / bits) when the stream was made with quals=True; lengths: [n] per-read lengths with lengths=True;
        n: reads of the batch (default: all rows of words).  The host arrays stay referenced until result(ticket)."""
        from .bam import pack_names
        w = self._host(words, torch.int32, "words")
        n = w.numel() // self.wpr if n is None else int(n)
        if w.numel() < n * self.wpr:
            raise ValueError("StreamingBam.submit: %d words for %d reads" % (w.numel(), n))
        if isinstance(names, tuple):
            nbytes, noff = names
        else:
            nbytes, noff = pack_names(names)
        nbytes = np.ascontiguousarray(nbytes, dtype=np.uint8)
        noff = np.ascontiguousarray(noff, dtype=np.uint32)
        want = n // 2 if self.pair is not None else n
        if noff.size != want + 1:
            raise ValueError("StreamingBam.submit: %d names for %d %s" % (noff.size - 1, want, "pairs" if self.pair is not None else "reads"))
        q = ln = None
        if quals is not None:
            q = self._host(quals, torch.uint8, "quals")
            if q.numel() < n * self.wpr * (32 // self.bits):
                raise ValueError("StreamingBam.submit: quals hold %d bytes for %d reads" % (q.numel(), n))
        if lengths is not None:
            ln = self._host(lengths, torch.int32, "lengths")
            if ln.numel() < n:
                raise ValueError("StreamingBam.submit: %d lengths for %d reads" % (ln.numel(), n))
        t = C.c_uint32(0)
        check(lib().nvb_pipeline_submit_bam(self._h, C.c_uint32(n), C.c_void_p(w.data_ptr()), C.c_void_p(q.data_ptr()) if q is not None else None,
                                            C.c_void_p(ln.data_ptr()) if ln is not None else None, C.c_void_p(nbytes.ctypes.data),
                                            C.c_void_p(noff.ctypes.data), C.byref(t)), "nvb_pipeline_submit_bam")
        self._keep[int(t.value)] = (w, q, ln, nbytes, noff)       # asynchronous copies: keep the sources alive until result()
        return int(t.value)

    def result(self, ticket: int):
        """wait for batch `ticket` and return its BamBatch (views of the pipeline's pinned host memory, valid until `depth` further
        submits)"""
        from ._lib import PipelineBamResultStruct
        from .bam import BamBatch
        r = PipelineBamResultStruct()
        check(lib().nvb_pipeline_wait_bam(self._h, C.c_uint32(ticket), C.byref(r)), "nvb_pipeline_wait_bam")
        self._keep.pop(ticket, None)
        self.last_device_ms = float(r.device_ms)
        nb = int(r.payload_bytes)
        payload = _host_view(r.payload, nb, torch.uint8) if nb else torch.empty(0, dtype=torch.uint8)
        ints = lambda ptr, k: tuple(int(v) for v in (C.c_uint32 * k).from_address(ptr))      # noqa: E731
        return BamBatch(payload=payload, compressed=self.compress, n_records=int(r.n_records), counts=ints(r.counts, 4),
                        n_hits=ints(r.n_hits, 3), n_rescue=ints(r.n_rescue, 2) if r.n_rescue else None, record_bytes=int(r.record_bytes),
                        n_blocks=int(r.n_blocks), device_ms=float(r.device_ms))

    def close(self):
        if self._h:
            lib().nvb_pipeline_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
