"""CPU: the BAI rules of nvb_bam_index, restated serially in tests/bai_oracle.py, against htslib's own index (bam_index_build) of the same
files: the sorted records of each synthetic case of tests/golden/make_bai_golden.py framed by write_bam's host path, replayed from
tests/golden/bai.npz and rebuilt live where oracle/_ref is built.  Bins are compared as sets (htslib writes them in hash order) and n_no_coor
per the deviation (htslib counts the first unplaced record only).  Argument validation of nvb_bam_sort / nvb_bam_index without a GPU."""
import ctypes as C
import os
import numpy as np
import pytest
from tests import bai_oracle as bo
from tests.golden.make_bai_golden import cases, frame, header, htslib_index, record, unmapped

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "bai.npz")
CASES = sorted(cases())


def _live():
    from oracle.ref_bai import RefBai
    return RefBai.available()


def check_against_htslib(recs, lens, header_bytes, block_offsets, hts: bytes):
    _, srt = bo.sort_records(recs)
    ours = bo.bai_bytes(srt, block_offsets, header_bytes, len(lens))
    a, a_no_coor, a_n = bo.parse_bai(ours)
    b, b_no_coor, b_n = bo.parse_bai(hts)
    assert a_n == b_n == len(lens)
    assert sorted(a) == sorted(b)
    for r in a:
        assert a[r][1] == b[r][1], ("linear index", r)
        assert set(a[r][0]) == set(b[r][0]), ("bins", r)
        for bin_ in a[r][0]:
            assert a[r][0][bin_] == [tuple(c) for c in b[r][0][bin_]], ("chunks", r, bin_)
    n_unplaced = sum(1 for x in srt if bo.sort_key(x)[0] == 0xFFFFFFFF)
    assert a_no_coor == n_unplaced
    assert b_no_coor == min(n_unplaced, 1)          # htslib stops counting after the first unplaced record
    return a


@pytest.mark.parametrize("case", CASES)
def test_rules_equal_htslib_golden(case):
    z = np.load(GOLDEN)
    recs = bo.split_records(z[case + "/records"].tobytes())
    lens = z[case + "/lens"].tolist()
    idx = check_against_htslib(recs, lens, int(z[case + "/header_bytes"]), z[case + "/block_offsets"], z[case + "/htslib_bai"].tobytes())
    if case == "deletion_levels":                   # records in bins of every level
        bins = {bo.rec_fields(r)[3] for r in recs}
        assert {sum(b >= f for f in (1, 9, 73, 585, 4681)) for b in bins} == {0, 1, 2, 3, 4, 5}
    if case == "dense_sparse":                      # merged upward, and apart
        bins = idx[0][0]
        assert any(len(c) > 1 for b, c in bins.items() if b != bo.META_BIN)
    if case == "many_contigs":
        assert 5 in idx and idx[5][1] == []          # only unmapped-placed records: no linear index


@pytest.mark.skipif(not _live(), reason="oracle/_ref is not built here")
@pytest.mark.parametrize("case", CASES)
def test_rules_equal_htslib_live(case):
    lens, recs = cases()[case]
    _, srt = bo.sort_records(recs)
    data, hb, offs = frame(header(lens), srt)
    check_against_htslib(recs, lens, hb, offs, htslib_index(data))
    if case == "block_boundary":                    # a record ends exactly at the first member's end
        assert 0xFF00 in np.cumsum([len(r) for r in srt])


def test_golden_replays_generator():
    """the golden file holds the records cases() makes now"""
    z = np.load(GOLDEN)
    for case in CASES:
        lens, recs = cases()[case]
        assert z[case + "/records"].tobytes() == b"".join(recs)
        assert z[case + "/lens"].tolist() == lens


def test_record_builder_fields():
    r = record("q", 3, 1000, flag=16, cigar=((0, 50), (2, 100_000), (0, 50)))
    assert bo.rec_fields(r) == (3, 1000, 1000 + 100_100, bo.reg2bin(1000, 101_100), True)
    assert bo.rec_fields(unmapped("u"))[:4] == (-1, -1, 0, 4680)


def test_argument_validation_without_gpu():
    """NULL arguments give NVB_E_INVALID (-1) and a contig longer than 2^29 NVB_E_UNSUPPORTED (-4), before any CUDA call; n = 0 sorts
    need no temp"""
    from nvbio_b200._lib import lib, BamSortOutStruct, BaiOutStruct
    L = lib()
    tb = C.c_size_t(0)
    so = BamSortOutStruct()
    assert L.nvb_bam_sort(None, None, C.c_uint32(4), C.byref(so), None, C.byref(tb), None) == -1           # no d_offsets
    so.d_offsets = 16
    assert L.nvb_bam_sort(None, None, C.c_uint32(4), C.byref(so), None, C.byref(tb), None) == -1           # no inputs
    assert L.nvb_bam_sort(C.c_void_p(16), C.c_void_p(16), C.c_uint32(4), None, None, C.byref(tb), None) == -1
    assert L.nvb_bam_sort(C.c_void_p(16), C.c_void_p(16), C.c_uint32(4), C.byref(so), None, None, None) == -1
    so.capacity = 64
    assert L.nvb_bam_sort(C.c_void_p(16), C.c_void_p(16), C.c_uint32(4), C.byref(so), None, C.byref(tb), None) == -1   # no d_records
    so.d_records = 24
    assert L.nvb_bam_sort(C.c_void_p(16), C.c_void_p(16), C.c_uint32(4), C.byref(so), None, C.byref(tb), None) == -1   # misaligned
    assert L.nvb_bam_sort(C.c_void_p(16), C.c_void_p(16), C.c_uint32(0x7FFFFFFF), C.byref(so), None, C.byref(tb), None) == -1
    bo_ = BaiOutStruct()

    def index(out=bo_, n=4, recs=16, offs=16, blocks=16, n_refs=2, max_len=1000, temp_bytes=tb):
        return L.nvb_bam_index(C.c_void_p(recs), C.c_void_p(offs), C.c_uint32(n), C.c_void_p(blocks), C.c_uint64(100), C.c_uint32(n_refs),
                               C.c_uint32(max_len), None if out is None else C.byref(out), None,
                               None if temp_bytes is None else C.byref(temp_bytes), None)
    assert index() == -1                                                                   # no d_size / d_status
    bo_.d_size, bo_.d_status = 16, 16
    assert index(out=None) == -1 and index(temp_bytes=None) == -1
    assert index(recs=None) == -1 and index(offs=None) == -1 and index(blocks=None) == -1
    assert index(n=0x7FFFFFFF) == -1 and index(n_refs=0x7FFFFFFF) == -1
    bo_.capacity = 100
    assert index() == -1                                                                   # no d_bai with a capacity
    bo_.capacity = 0
    assert index(max_len=(1 << 29) + 1) == -4
    assert index(max_len=(1 << 29) + 1, recs=None) == -1                                  # a failed check wins over it
