"""CPU: the MAPQ of nvb_seed_extend_mapq (bowtie_mapq2 in pipeline_core.cuh, compiled for the host by tests/host/mapq_harness.cu), its
Python restatement and the MapqParams --score-min helper against nvBowtie's own BowtieMapq2 and SimpleFunc (tests/golden/mapq.npz,
written from the reference by tests/golden/make_mapq_golden.py), and the entry point's argument validation."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle.ref_mapq import RefMapq
from tests.golden.make_mapq_golden import mapq_grid, SIMPLE_FUNCS
from tests.mapq_oracle import bowtie_mapq2

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "mapq.npz")
SO = os.path.join(HERE, "host", "libmapq_harness.so")
SRC = os.path.join(HERE, "host", "mapq_harness.cu")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def G():
    return np.load(GOLDEN)


def grid_points(G):
    """every fixture point as flat arrays (best, has_second, second, length, match_bonus, min_score) and the fixture's MAPQ"""
    cols = [[] for _ in range(6)]
    for length, bonus, ms, _ in G["cfg"]:
        best, has, second = mapq_grid(length, bonus, ms)
        for c, v in zip(cols, (best, has, second, np.full(len(best), length, np.uint32), np.full(len(best), bonus, np.int32),
                               np.full(len(best), ms, np.int32))):
            c.append(v)
    return [np.concatenate(c) for c in cols], G["mapq"]


def test_fixture_covers_the_grid(G):
    assert G["offsets"][-1] == len(G["mapq"])
    for c, (length, bonus, ms, _) in enumerate(G["cfg"]):
        assert G["offsets"][c + 1] - G["offsets"][c] == len(mapq_grid(length, bonus, ms)[0])
    assert {int(v) for v in G["cfg"][:, 0]} == {1, 20, 50, 100, 150, 151, 250, 1000}
    assert {int(v) for v in G["cfg"][:, 1]} == {0, 2, 3}
    # both branches of BowtieMapq2, with and without a second alignment, take most of their values
    assert len(np.unique(G["mapq"])) >= 40


def test_host_build_equals_reference(G):
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    H = C.CDLL(SO)
    (best, has, second, length, bonus, ms), want = grid_points(G)
    got = np.zeros(len(best), np.uint8)
    H.hh_bowtie_mapq2(_p(best), _p(has), _p(second), _p(length), _p(bonus), _p(ms), C.c_uint32(len(best)), _p(got))
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(best[i]), int(has[i]), int(second[i]), int(length[i]), int(bonus[i]), int(ms[i]), int(got[i]), int(want[i])) for i in bad[:5]]


def test_python_restatement_equals_reference(G):
    (best, has, second, length, bonus, ms), want = grid_points(G)
    got = bowtie_mapq2(best, has, second, length, bonus, ms)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(best[i]), int(has[i]), int(second[i]), int(length[i]), int(bonus[i]), int(ms[i]), int(got[i]), int(want[i])) for i in bad[:5]]
    # a read without an alignment (INT_MIN) gets 0 whatever the rest
    assert not bowtie_mapq2(np.full(4, -2**31), [0, 1, 0, 1], -2**31, 150, [0, 0, 2, 2], [-90, -90, 50, 50]).any()


def test_simple_func_helper_equals_reference(G):
    from nvbio_b200.pipeline import simple_func
    x = G["sf_x"]
    for (code, k, m), want in zip(G["sf_funcs"], G["sf_vals"]):
        kind = "LGS"[int(code)]
        assert np.array_equal(simple_func(kind, k, m, x), want), (kind, k, m)
    # the min scores of the MAPQ grid are the same functions
    for length, bonus, ms, f in G["cfg"]:
        kind, k, m = SIMPLE_FUNCS[int(f)]
        assert int(simple_func(kind, k, m, [length])[0]) == ms


def test_mapq_params_presets():
    import torch
    from nvbio_b200.pipeline import MapqParams, simple_func
    p = MapqParams.local(250, device="cpu")
    assert p.match_bonus == 2 and p.max_read_len == 250 and p.min_score.dtype == torch.int32
    assert int(p.min_score[150]) == int(10.0 * np.log(150)) == 50
    assert int(p.min_score[0]) == -(2**31 - 1)                      # log(0) = -inf, clamped above INT_MIN
    e = MapqParams.end_to_end(150, device="cpu")
    assert e.match_bonus == 0 and int(e.min_score[150]) == -90 and int(e.min_score[0]) == 0
    with pytest.raises(ValueError):
        simple_func("X", 0.0, 1.0, [1])


@pytest.mark.skipif(not RefMapq.available(), reason="oracle/_ref/libnvbio_ref_mapq.so (the reference's own code) is not built here")
def test_fixture_equals_live_reference(G):
    R = RefMapq()
    (best, has, second, length, bonus, ms), want = grid_points(G)
    assert np.array_equal(R.mapq(best, has, second, length, bonus, ms), want)
    for (code, k, m), vals in zip(G["sf_funcs"], G["sf_vals"]):
        assert np.array_equal(R.simple_func("LGS"[int(code)], k, m, G["sf_x"]), vals)


def test_argument_validation_without_gpu():
    """nvb_seed_extend_mapq rejects missing MAPQ inputs / outputs and a min-score table shorter than the reads with NVB_E_INVALID (-1)
    before any CUDA call, also when the reads would be NVB_E_UNSUPPORTED (-4)"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, SeedExtendParamsStruct, FmIndexStruct, MapqParamsStruct,
                                 MapqOutStruct, BestAlignmentOutStruct)
    L = _lib.lib()
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    tb = C.c_size_t(0)

    def call(mp, mo, reads=ss, ba=None, params=sp):
        r = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return L.nvb_seed_extend_mapq(C.byref(fm), C.c_void_p(16), r(reads), C.c_uint32(8), C.byref(params), C.c_uint32(100),
                                      C.c_void_p(16), C.c_void_p(16), None, None, None, None, None, r(ba), r(mp), r(mo), None, C.byref(tb), None)

    def good():
        mp = MapqParamsStruct(); mp.d_min_score, mp.max_read_len, mp.match_bonus = 16, 150, 2
        mo = MapqOutStruct(); mo.d_second_score, mo.d_mapq = 16, 16
        return mp, mo

    mp, mo = good()
    assert call(None, mo) == -1 and call(mp, None) == -1 and call(None, None) == -1
    for field in ("d_min_score",):
        mp, mo = good(); setattr(mp, field, None); assert call(mp, mo) == -1
    for field in ("d_second_score", "d_mapq"):
        mp, mo = good(); setattr(mo, field, None); assert call(mp, mo) == -1
    mp, mo = good(); mp.max_read_len = 149
    assert call(mp, mo) == -1
    mp, mo = good(); assert call(mp, mo, reads=None) == -1
    # 8-bit reads are NVB_E_UNSUPPORTED (-4), but every failed MAPQ or best-alignment check wins over it
    s8 = StringSetStruct(); s8.d_words = 16; s8.bits = 8; s8.big_endian = 1; s8.stride = 152; s8.length = 150
    mp, mo = good(); assert call(mp, mo, reads=s8) == -4
    mp, mo = good(); mp.max_read_len = 149; assert call(mp, mo, reads=s8) == -1
    mp, mo = good(); mo.d_mapq = None; assert call(mp, mo, reads=s8) == -1
    mp, mo = good(); assert call(None, mo, reads=s8) == -1 and call(mp, None, reads=s8) == -1
    ba = BestAlignmentOutStruct(); ba.d_ops = 16; ba.max_ops = 0; ba.d_n_ops = 16; ba.d_begin = 16
    mp, mo = good(); assert call(mp, mo, ba=ba) == -1 and call(mp, mo, reads=s8, ba=ba) == -1
    # the paired traceback's 512 bp limit does not apply to a single-end traceback: reads of 513 bp reach the seed checks
    s513 = StringSetStruct(); s513.d_words = 16; s513.bits = 2; s513.big_endian = 1; s513.stride = 528; s513.length = 513
    no_seed = SeedExtendParamsStruct(); no_seed.seed_len, no_seed.seed_interval, no_seed.band_len, no_seed.type = 0, 10, 31, 1
    no_seed.both_strands, no_seed.max_seed_hits, no_seed.dedup_jobs, no_seed.scheme = 1, 100, 1, sch
    ba.max_ops = 1100
    mp, mo = good(); mp.max_read_len = 513; assert call(mp, mo, reads=s513, ba=ba, params=no_seed) == -1
