"""CPU: the selection rule of nvb_seed_extend_all (reportable / make_best_key / select_distinct in pipeline_core.cuh, compiled for the host
by tests/host/all_harness.cu) against its restatement (tests/all_oracle.py) on seeded random candidate lists, and the entry point's
argument validation."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from tests.all_oracle import select
from tests.pipeline_oracle import EMPTY_SINK

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "liball_harness.so")
SRC = os.path.join(HERE, "host", "all_harness.cu")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    h = C.CDLL(SO)
    h.hh_select_all.restype = C.c_uint32
    return h


def host_select(H, score, tie, end, strand, sink_x, length, min_score, k):
    n = len(score)
    out = np.zeros(max(n, 1), np.uint32)
    a = [np.ascontiguousarray(score, np.int32), np.ascontiguousarray(tie, np.uint32), np.ascontiguousarray(end, np.uint32),
         np.ascontiguousarray(strand, np.uint8), np.ascontiguousarray(sink_x, np.uint32)]
    m = H.hh_select_all(C.c_uint32(n), *[_p(x) for x in a], C.c_uint32(length), C.c_int32(min_score), C.c_uint32(k), _p(out))
    return [int(v) for v in out[:m]]


def candidates(rng, kind, length):
    """one read's candidate list of a given flavour"""
    n = int(rng.integers(1, 40)) if kind != "large" else int(rng.integers(200, 600))
    d = length // 2
    if kind == "near0":                                     # ends near position 0: the min(bp, len/2) clamp
        end = rng.integers(0, 2 * length, n)
    elif kind == "spaced":                                  # ends exactly len/2 (and len/2 + 1) apart
        end = 5000 + d * rng.integers(0, 8, n) + rng.integers(0, 2, n)
    else:
        end = rng.integers(0, 50 * length, n)
    score = rng.integers(40, 60, n) if kind != "ties" else rng.integers(50, 52, n)
    tie = rng.permutation(10 * n)[:n]                        # unique, as both paths' tie indices are
    strand = rng.integers(0, 2, n)
    if kind == "both_strands":                               # equal ends on both strands
        end[1::2] = end[0::2][:len(end[1::2])]
    sink_x = np.where(rng.random(n) < 0.1, EMPTY_SINK, 1)    # empty jobs
    return score, tie, end, strand, sink_x


@pytest.mark.parametrize("k", [1, 2, 5, 0, 1000])
def test_select_equals_restatement(H, k):
    rng = np.random.default_rng(11 + k)
    seen = dict(multi=0, cut=0)
    for it in range(600):
        kind = ["random", "ties", "near0", "spaced", "both_strands", "large"][it % 6]
        length = int(rng.choice([1, 2, 3, 50, 100, 101, 150, 512]))
        score, tie, end, strand, sink_x = candidates(rng, kind, length)
        ms = int(rng.choice([0, 50, int(np.median(score))]))          # the min-score boundary: scores equal to it are candidates
        want = select(score, tie, end, strand, sink_x, length, ms, k)
        got = host_select(H, score, tie, end, strand, sink_x, length, ms, k)
        assert got == want, (it, kind, length, ms)
        seen["multi"] += len(want) > 1
        seen["cut"] += k > 0 and len(want) == k
    assert seen["multi"] > 50 or k == 1
    assert seen["cut"] > 50 or k in (0, 1000)


def test_select_rules(H):
    """hand-made lists: ties by tie index, the len/2 distance in both directions, the clamp near 0, strands, min score, empty jobs, k"""
    L = 100
    s = lambda *a, **kw: host_select(H, *a, **kw)          # noqa: E731
    # equal scores: the smaller tie index ranks first; the other end is within len/2: not distinct
    assert s([50, 50], [7, 3], [1000, 1050], [0, 0], [1, 1], L, 0, 0) == [1]
    assert s([50, 50], [7, 3], [1000, 1051], [0, 0], [1, 1], L, 0, 0) == [1, 0]
    assert s([50, 50], [7, 3], [1000, 949], [0, 0], [1, 1], L, 0, 0) == [1, 0]
    assert s([50, 50], [7, 3], [1000, 950], [0, 0], [1, 1], L, 0, 0) == [1]
    # the same end on the other strand is distinct
    assert s([50, 49], [0, 1], [1000, 1000], [0, 1], [1, 1], L, 0, 0) == [0, 1]
    # near position 0 the window is [bp - min(bp, len/2), bp + len/2]
    assert s([50, 49], [0, 1], [10, 0], [0, 0], [1, 1], L, 0, 0) == [0]
    assert s([50, 49], [0, 1], [10, 61], [0, 0], [1, 1], L, 0, 0) == [0, 1]
    # distinct from EVERY admitted one: c is far from a but close to b
    assert s([60, 55, 50], [0, 1, 2], [1000, 2000, 2040], [0, 0, 0], [1, 1, 1], L, 0, 0) == [0, 1]
    # min score: equal qualifies, below does not; empty jobs never
    assert s([50, 49, 70], [0, 1, 2], [0, 5000, 9000], [0, 0, 0], [1, 1, EMPTY_SINK], L, 50, 0) == [0]
    # k: 1 gives the best, a large k every distinct one
    assert s([50, 60, 55], [0, 1, 2], [0, 5000, 9000], [0, 0, 0], [1, 1, 1], L, 0, 1) == [1]
    assert s([50, 60, 55], [0, 1, 2], [0, 5000, 9000], [0, 0, 0], [1, 1, 1], L, 0, 9) == [1, 2, 0]
    assert s([], [], [], [], [], L, 0, 0) == []


def test_argument_validation_without_gpu():
    """nvb_seed_extend_all rejects missing structs and outputs, a best_alignment, max_ops 0 and a short min-score table with NVB_E_INVALID
    (-1), and reads over 512 bp with NVB_E_UNSUPPORTED (-4), before any CUDA call"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, SeedExtendParamsStruct, FmIndexStruct, MapqParamsStruct,
                                 MapqOutStruct, BestAlignmentOutStruct, AllParamsStruct, AllOutStruct)
    L = _lib.lib()
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    tb = C.c_size_t(0)

    def good():
        mp = MapqParamsStruct(); mp.d_min_score, mp.max_read_len, mp.match_bonus = 16, 150, 2
        mo = MapqOutStruct(); mo.d_second_score, mo.d_mapq = 16, 16
        ap = AllParamsStruct(); ap.max_per_read, ap.capacity = 2, 100
        ao = AllOutStruct(); ao.d_first = ao.d_read = ao.d_score = ao.d_pos = ao.d_count = 16
        ao.alignment.d_ops, ao.alignment.max_ops, ao.alignment.d_n_ops, ao.alignment.d_begin, ao.alignment.d_strand = 16, 331, 16, 16, 16
        return mp, mo, ap, ao

    def call(mp, mo, ap, ao, reads=ss, ba=None):
        r = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return L.nvb_seed_extend_all(C.byref(fm), C.c_void_p(16), r(reads), C.c_uint32(8), C.byref(sp), C.c_uint32(100),
                                     C.c_void_p(16), C.c_void_p(16), None, None, None, None, None, r(ba), r(mp), r(mo), r(ap), r(ao),
                                     None, C.byref(tb), None)

    mp, mo, ap, ao = good()
    assert call(mp, mo, ap, ao) not in (-1, -4)                             # passes validation (a size query where there is a device)
    assert call(None, mo, ap, ao) == -1 and call(mp, None, ap, ao) == -1
    assert call(mp, mo, None, ao) == -1 and call(mp, mo, ap, None) == -1
    for f in ("d_first", "d_read", "d_score", "d_pos", "d_count"):
        mp, mo, ap, ao = good(); setattr(ao, f, None); assert call(mp, mo, ap, ao) == -1, f
    for f in ("d_ops", "d_n_ops", "d_begin", "d_strand"):
        mp, mo, ap, ao = good(); setattr(ao.alignment, f, None); assert call(mp, mo, ap, ao) == -1, f
    mp, mo, ap, ao = good(); ao.alignment.max_ops = 0; assert call(mp, mo, ap, ao) == -1
    mp, mo, ap, ao = good(); mp.max_read_len = 149; assert call(mp, mo, ap, ao) == -1
    mp, mo, ap, ao = good(); mo.d_mapq = None; assert call(mp, mo, ap, ao) == -1
    ba = BestAlignmentOutStruct(); ba.d_ops = 16; ba.max_ops = 331; ba.d_n_ops = 16; ba.d_begin = 16; ba.d_strand = 16
    mp, mo, ap, ao = good(); assert call(mp, mo, ap, ao, ba=ba) == -1
    s513 = StringSetStruct(); s513.d_words = 16; s513.bits = 2; s513.big_endian = 1; s513.stride = 528; s513.length = 513
    mp, mo, ap, ao = good(); mp.max_read_len = 513; assert call(mp, mo, ap, ao, reads=s513) == -4
    mp, mo, ap, ao = good(); mp.max_read_len = 512
    s512 = StringSetStruct(); s512.d_words = 16; s512.bits = 2; s512.big_endian = 1; s512.stride = 512; s512.length = 512
    assert call(mp, mo, ap, ao, reads=s512) not in (-1, -4)                 # 512 bp is supported


# ---- BAM records of several alignments per read (nvb_bam_records_all) -------------------------------------------------------------------

from tests.test_bam_host import traced_inputs, HF, genome, LIVE            # noqa: E402,F401  (HF, genome: fixtures)
from tests.all_oracle import all_records                                   # noqa: E402


@pytest.fixture(scope="module")
def HB():
    so = os.path.join(HERE, "host", "libbam_all_harness.so")
    src = os.path.join(HERE, "host", "bam_all_harness.cu")
    deps = [src] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("bam_core.cuh", "finish_core.cuh", "pipeline_core.cuh", "fm_core.cuh",
                                                                               "common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", so, src])
    h = C.CDLL(so)
    h.hh_bam_all.restype = C.c_uint32
    return h


def all_inputs(HF, rng, genome, bits, quals, mapq):
    """several alignments per read from a traced batch: read r's alignments are copies of traced alignment r at shifted begins (some
    across contig cuts or past the genome), unaligned or unfinished copies among them; first / capacity as nvb_seed_extend_all writes them"""
    base = traced_inputs(HF, rng, genome, bits, False, n_reads=120, quals=quals, mapq=mapq)
    n = len(base["reads"])
    per = rng.integers(0, 6, n)
    first = np.concatenate([[0], np.cumsum(per)]).astype(np.uint32)
    src = np.repeat(np.arange(n), per)
    A = len(src)
    inp = dict(base)
    for f in ("n_ops", "begin", "strand", "cigar", "n_cigar", "md", "md_len", "edits"):
        inp[f] = np.ascontiguousarray(base[f][src])
    G = int(base["contig_begin"][-1])
    shift = np.where(rng.random(A) < 0.5, 0, rng.integers(-3000, 3000, A))
    inp["begin"][:, 0] = np.clip(inp["begin"][:, 0].astype(np.int64) + shift, 0, G + 10).astype(np.uint32)
    inp["n_ops"][rng.random(A) < 0.1] = 0
    inp["edits"][rng.random(A) < 0.05, 0] = 0xFFFFFFFF
    inp["score"] = rng.integers(-300, 300, A).astype(np.int32)
    inp["strand"] = rng.integers(0, 2, A).astype(np.uint8)
    return inp, first


def run_all_host(HB, inp, first, capacity, bits):
    from nvbio_b200._lib import BamAllInStruct
    from nvbio_b200.strings import pack_symbols
    n = len(inp["reads"])
    keep = []

    def arr(x, dt):
        if x is None:
            return None
        y = np.ascontiguousarray(np.asarray(x).astype(dt))
        keep.append(y)
        return y.ctypes.data
    lens = np.array([len(r) for r in inp["reads"]], np.uint32)
    offs = (np.concatenate([[0], np.cumsum(lens)[:-1]])).astype(np.uint32)
    words = pack_symbols(np.concatenate(list(inp["reads"]) + [np.zeros(1, np.uint8)]), bits, True); keep.append(words)
    a = BamAllInStruct()
    b = a.base
    b.reads.d_words, b.reads.bits, b.reads.big_endian = words.ctypes.data, bits, 1
    b.reads.d_offsets, b.reads.d_lengths, b.reads.length = arr(offs, np.uint32), arr(lens, np.uint32), int(lens.max())
    if inp["quals"] is not None:
        b.d_read_quals = arr(np.concatenate([np.asarray(x, np.uint8) for x in inp["quals"]] + [np.zeros(1, np.uint8)]), np.uint8)
    b.d_n_ops, b.d_begin, b.d_strand = arr(inp["n_ops"], np.uint32), arr(inp["begin"], np.uint32), arr(inp["strand"], np.uint8)
    f = b.finish
    f.d_cigar, f.max_cigar, f.d_n_cigar = arr(inp["cigar"], np.uint32), inp["cigar"].shape[1], arr(inp["n_cigar"], np.uint32)
    f.d_md, f.max_md, f.d_md_len, f.d_edits = arr(inp["md"], np.uint8), inp["md"].shape[1], arr(inp["md_len"], np.uint32), arr(inp["edits"], np.uint32)
    b.d_score, b.d_mapq, b.d_second_score = arr(inp["score"], np.int32), arr(inp["mapq"], np.uint8), arr(inp["second"], np.int32)
    b.d_contig_begin, b.n_contigs = arr(inp["contig_begin"], np.uint32), len(inp["contig_begin"]) - 1
    nb = [nm.encode() for nm in inp["names"]]
    b.d_names = arr(np.frombuffer(b"".join(nb) + b"\0", np.uint8), np.uint8)
    b.d_name_offsets = arr(np.concatenate([[0], np.cumsum([len(x) for x in nb])]), np.uint32)
    a.d_first, a.capacity = arr(first, np.uint32), int(capacity)
    slots = n + int(capacity)
    buf = np.zeros(slots * (400 + 4 * inp["cigar"].shape[1] + inp["md"].shape[1]) + 16, np.uint8)
    o = np.zeros(slots + 1, np.uint64); cnt = np.zeros(4, np.uint32)
    k = HB.hh_bam_all(C.byref(a), C.c_uint32(n), _p(buf), _p(o), _p(cnt))
    return [buf[int(o[i]):int(o[i + 1])].tobytes() for i in range(k)], o, cnt


@pytest.mark.parametrize("bits", [2, 4])
def test_all_records_layout(HB, HF, genome, bits):
    """FLAG, MAPQ, XS on the primary only, NH, the primary choice when rank 0 is unplaceable, one unmapped record per read without a
    placeable alignment or beyond the capacity: the host build of the planning and compose routines against the restatement"""
    from oracle.ref_bam import RefBam
    from tests import bam_oracle as bo
    rng = np.random.default_rng(40 + bits)
    seen = dict(secondary=0, primary_not_rank0=0, unmapped_with_alignments=0, beyond=0)
    for i in range(4):
        inp, first = all_inputs(HF, rng, genome, bits, quals=i % 2 == 0, mapq=i != 3)
        A = int(first[-1])
        capacity = A if i % 2 == 0 else int(first[len(first) // 2])
        want, cnt = all_records(inp, first, capacity)
        got, o, gcnt = run_all_host(HB, inp, first, capacity, bits)
        assert list(gcnt) == cnt
        assert len(got) == len(want)
        for k, (g, (w, sam)) in enumerate(zip(got, want)):
            assert g == w, (k, sam)
        assert (o[len(got):] == o[len(got)]).all()                       # entries past the records repeat the total
        flags = [int.from_bytes(w[18:20], "little") for w, _ in want]
        seen["secondary"] += sum(f & 0x100 != 0 for f in flags)
        seen["beyond"] += cnt[3]
        for r in range(len(inp["reads"])):
            if first[r + 1] <= capacity and first[r + 1] > first[r]:
                st = [bo.place(inp, a)[0] for a in range(first[r], first[r + 1])]
                seen["primary_not_rank0"] += st[0] != 1 and 1 in st
                seen["unmapped_with_alignments"] += 1 not in st
        # exactly one non-secondary record per read
        assert sum(f & 0x100 == 0 for f in flags) == len(inp["reads"])
        if LIVE and RefBam.available():
            header = bo.header_text(inp["contig_names"], inp["contig_lengths"])
            assert RefBam().encode(header, [s for _, s in want]) == [w for w, _ in want]
    assert all(v > 0 for v in seen.values()), seen


def test_bam_records_all_argument_validation_without_gpu():
    from nvbio_b200 import _lib
    from nvbio_b200._lib import BamAllInStruct, BamOutStruct
    L = _lib.lib()
    tb = C.c_size_t(0)

    def good():
        a = BamAllInStruct(); b = a.base
        b.reads.d_words, b.reads.bits, b.reads.big_endian, b.reads.stride, b.reads.length = 16, 2, 1, 160, 150
        b.d_n_ops = b.d_begin = b.d_strand = b.d_score = b.d_contig_begin = b.d_names = b.d_name_offsets = 16
        b.n_contigs = 1
        f = b.finish
        f.d_cigar = f.d_n_cigar = f.d_md = f.d_md_len = f.d_edits = 16; f.max_cigar, f.max_md = 10, 10
        a.d_first, a.capacity = 16, 100
        o = BamOutStruct(); o.d_records, o.capacity, o.d_offsets, o.d_counts = 16, 4096, 16, 16
        return a, o
    call = lambda a, o, n=8: L.nvb_bam_records_all(C.byref(a) if a is not None else None, C.c_uint32(n), C.byref(o), None, C.byref(tb), None)  # noqa: E731
    a, o = good(); assert call(a, o) not in (-1, -4)
    assert call(None, o) == -1
    a, o = good(); a.d_first = None; assert call(a, o) == -1
    a, o = good(); a.base.d_pair_flags = 16; assert call(a, o) == -1
    a, o = good(); a.base.finish.d_edits = None; assert call(a, o) == -1
    a, o = good(); o.d_records = 24; assert call(a, o) == -1                  # misaligned
    a, o = good(); a.capacity = 0x7FFFFFF8; assert call(a, o) == -1
