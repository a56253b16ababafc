"""The closed-form index of T = A^F . R (tests/long_genome.py) against the oracle's suffix sort of T itself, at sizes the oracle can
sort: suffix array, primary row, stored BWT, sampled SA and the device builders' words (run on host tensors here), with F below, at
and above the longest A-run of R and A-runs planted inside R; the row map between two such genomes and the closed-form range sizes
of A^s and A^s . R[:q] against the oracle's match(); and the length limits of ContigTable and the C ABI."""
import ctypes as C
import numpy as np
import pytest

from oracle import orc
from nvbio_b200.strings import pack_symbols
from tests.long_genome import LongGenome, a_runs, device_bwt, device_genome, device_sa


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


def _random_R(r, seed, plant=((100, 20), (1500, 7), (2500, 3))):
    """random symbols with non-A ends and A-runs of the planted (position, length)s"""
    rng = np.random.default_rng(seed)
    R = rng.integers(0, 4, r).astype(np.uint8)
    for p, ln in plant:
        R[p:p + ln] = 0
        R[p + ln] = 1 + (p % 3)
    R[0], R[-1] = 2, 3
    return R


@pytest.fixture(scope="module")
def R_and_sa(O):
    R = _random_R(3000, 11)
    return R, O.build_index(R).sa


def test_a_runs():
    R = np.array([1, 0, 0, 0, 2, 0, 3, 0, 0, 1], np.uint8)
    assert a_runs(R).tolist() == [0, 3, 2, 1, 0, 1, 0, 2, 1, 0]


@pytest.mark.parametrize("F", [1, 3, 7, 19, 20, 21, 40, 1000, 5000])
def test_construction_matches_oracle(O, R_and_sa, F):
    R, sa_R = R_and_sa
    lg = LongGenome(R, F, sa_R)
    assert lg.m == 20
    text = lg.text()
    ref = O.build_index(text)
    assert np.array_equal(lg.sa(), ref.sa.astype(np.int64))
    assert lg.primary == ref.primary
    assert np.array_equal(pack_symbols(lg.bwt(), pad_words=0), ref.bwt[:(lg.n + 15) // 16])
    # the device builders' words, made here on host tensors
    bw = device_bwt(lg, "cpu").numpy().view(np.uint32)
    assert np.array_equal(bw, ref.bwt)
    sa = device_sa(lg, "cpu").numpy().view(np.uint32)
    want = ref.sa.astype(np.uint32)
    want[0] = 0xFFFFFFFF
    assert np.array_equal(sa, want)
    assert np.array_equal(sa[::16], ref.ssa)
    gw = device_genome(lg, "cpu").numpy().view(np.uint32)
    pk = pack_symbols(text, pad_words=0)
    assert np.array_equal(gw[:len(pk)], pk) and not gw[len(pk):].any()
    # occ table and L2 of the closed-form BWT equal the oracle's (the same words give the same table)
    idx = O.index_from_sa(text, lg.sa().astype(np.int32))
    assert np.array_equal(idx.bwt_occ, ref.bwt_occ) and np.array_equal(idx.L2, ref.L2) and np.array_equal(idx.ssa, ref.ssa)


def _queries(R, rng, n, ln):
    pos = rng.integers(0, len(R) - ln, n)
    return np.stack([R[p:p + ln] for p in pos])


def _match(O, idx, qs):
    qs = [np.asarray(q, np.uint8) for q in qs]
    lens = np.array([len(q) for q in qs])
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    out, _ = O.match(idx, np.concatenate(qs), off, lens)
    return out.astype(np.int64)


def test_row_map_and_closed_form_ranges(O, R_and_sa):
    """ranges on A^F2 . R = ranges on A^F1 . R moved by F2 - F1 (non-empty ranges of queries that hold a non-A), A^s = rows
    1 .. a_run_range_size(s), and A^s . R[:q] has boundary_range_size(s, q) rows"""
    R, sa_R = R_and_sa
    rng = np.random.default_rng(5)
    small, big = LongGenome(R, 40, sa_R), LongGenome(R, 3000, sa_R)
    d = big.shift(small)
    i1, i2 = O.build_index(small.text()), O.build_index(big.text())
    qs = list(_queries(R, rng, 300, 12)) + list(_queries(R, rng, 300, 5)) + [R[95:130], R[1490:1520], R[:30]]
    r1, r2 = _match(O, i1, qs), _match(O, i2, qs)
    ne = r1[:, 0] <= r1[:, 1]
    assert ne.sum() > 300
    assert np.array_equal(ne, r2[:, 0] <= r2[:, 1])
    ne &= np.array([q.any() for q in qs])                  # A's alone: see below
    assert np.array_equal(r1[ne] + d, r2[ne])
    # suffix array positions move with the rows
    s1, s2 = small.sa(), big.sa()
    assert np.array_equal(s1[1:] + d, s2[1 + d:])
    for lg, idx in ((small, i1), (big, i2)):
        for s in (1, 2, 3, 7, 12, 20, 21, 40, 45):
            (x, y), = _match(O, idx, [np.zeros(s, np.uint8)])
            size = lg.a_run_range_size(s)
            assert (x, y) == (1, size) if size else x > y, s
        for s in (1, 3, 7, 20, 39, 40, 41):
            for q in (1, 2, 5, 20):
                (x, y), = _match(O, idx, [np.concatenate([np.zeros(s, np.uint8), R[:q]])])
                assert max(y - x + 1, 0) == lg.boundary_range_size(s, q), (s, q)


def test_contig_table_limits():
    """a contig of 2^31 bases or more has no BAM position (int32 POS and l_ref); a genome longer than 2^32 - 2 has no index"""
    from nvbio_b200.bam import ContigTable
    with pytest.raises(ValueError):
        ContigTable(["a"], [1 << 31])
    with pytest.raises(ValueError):
        ContigTable(["a", "b"], [100, 1 << 31])
    assert ContigTable(["a", "b"], [(1 << 31) - 1, (1 << 31) - 1]).genome_len == 0xFFFFFFFE      # the longest index text
    with pytest.raises(ValueError):
        ContigTable(["a", "b", "c"], [(1 << 31) - 1, (1 << 31) - 1, 1])


def test_fm_length_limit_without_gpu():
    """texts longer than NVB_FM_MAX_LENGTH = 2^32 - 2 are refused (NVB_E_INVALID) before any CUDA call: by every entry point that takes
    an index, by the occ build and by the suffix sort"""
    from nvbio_b200 import _lib
    from nvbio_b200.fmindex import MAX_LENGTH
    assert MAX_LENGTH == 0xFFFFFFFE
    L = _lib.lib()
    tb = C.c_size_t(0)
    L2 = (C.c_uint32 * 5)()
    assert L.nvb_fm_build_occ(C.c_void_p(32), C.c_uint32(0xFFFFFFFF), C.c_void_p(32), L2, None, C.byref(tb), None) == -1
    prim = C.c_uint32(0)
    assert L.nvb_fm_build_bwt(C.c_void_p(32), C.c_uint32(0xFFFFFFFF), C.c_void_p(32), C.byref(prim), C.c_void_p(32), C.c_uint32(16), None,
                              None, C.byref(tb), None) == -1
    s = _lib.FmIndexStruct()
    s.d_bwt_occ, s.length, s.primary = 32, 0xFFFFFFFF, 1
    assert L.nvb_fm_rank(C.byref(s), C.c_void_p(32), C.c_void_p(32), C.c_uint32(1), C.c_void_p(32), None) == -1
