"""CPU: the reseeding rules of nvb_seed_extend_reseed (reseed_offset / reseed_read, nvbio_b200/csrc/pipeline_core.cuh), compiled for
the host by tests/host/reseed_harness.cu, against tests/reseed_oracle.py at their edges."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from tests import reseed_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "libreseed_harness.so")
SRC = os.path.join(HERE, "host", "reseed_harness.cu")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("pipeline_core.cuh", "fm_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Wno-deprecated-declarations",
                               "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    return C.CDLL(SO)


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def host_flags(H, s, c, rep, aligned):
    s, c, rep = u32(s), u32(c), u32(rep)
    al = np.ascontiguousarray(aligned, dtype=np.uint8)
    out = np.zeros(len(s), np.uint8)
    H.rh_reseed_read(_p(s), _p(c), _p(rep), _p(al), C.c_uint32(len(s)), _p(out))
    return out


def test_flag_rule_edges(H):
    """range_count 0, equality at rep_seeds * range_count, one below it, uint32 wrap of the product and of the sum, unaligned reads"""
    rows = [
        (0, 0, 300, 1), (0, 0, 0, 1),                        # no range: flagged whatever rep_seeds
        (600, 2, 300, 1), (599, 2, 300, 1), (601, 2, 300, 1),  # mean exactly rep_seeds / just below / above
        (5, 3, 0x55555556, 1),                               # 3 * 0x55555556 wraps to 2: 5 >= 2
        (1, 3, 0x55555556, 1),                               # ... and 1 < 2
        (0xFFFFFFFF, 1, 0xFFFFFFFF, 1), (0xFFFFFFFE, 1, 0xFFFFFFFF, 1),
        ((0xFFFFFFFF + 5) & 0xFFFFFFFF, 2, 8, 1),            # a wrapped sum: 4 < 16
        (3, 3, 8, 1), (3, 3, 8, 0), (0, 0, 8, 0), (100, 2, 8, 0),
    ]
    s, c, rep, al = (np.array(v, np.int64) for v in zip(*rows))
    want = np.array([ro.reseed_flag(int(a), int(b), int(r), bool(x)) for a, b, r, x in rows], np.uint8)
    assert np.array_equal(host_flags(H, s, c, rep, al), want)
    assert list(want) == [1, 1, 1, 0, 1, 1, 0, 1, 0, 0, 0, 1, 1, 1]


def test_flag_rule_random(H):
    rng = np.random.default_rng(7)
    n = 20000
    s = rng.integers(0, 2**32, n, dtype=np.uint64); c = rng.integers(0, 40, n); rep = rng.integers(0, 2**32, n, dtype=np.uint64)
    small = rng.random(n) < 0.5
    s[small] = rng.integers(0, 4000, small.sum()); rep[small] = rng.integers(0, 300, small.sum())
    al = rng.integers(0, 2, n)
    want = np.array([ro.reseed_flag(int(a), int(b), int(r), bool(x)) for a, b, r, x in zip(s, c, rep, al)], np.uint8)
    assert np.array_equal(host_flags(H, s, c, rep, al), want)


@pytest.mark.parametrize("max_reseed", [0, 1, 2, 3])
@pytest.mark.parametrize("interval", [1, 3, 4, 10, 13, 24])
def test_offsets(H, max_reseed, interval):
    """o_r = r * floor(I / (max_reseed + 1)): also for intervals that are not a multiple of max_reseed + 1"""
    r = np.arange(max_reseed + 1)
    out = np.zeros(len(r), np.uint32)
    H.rh_reseed_offset(_p(u32(r)), _p(u32(np.full(len(r), interval))), _p(u32(np.full(len(r), max_reseed))), C.c_uint32(len(r)), _p(out))
    want = [ro.reseed_offset(int(k), interval, max_reseed) for k in r]
    assert list(out) == want
    assert want[0] == 0 and all(w < interval for w in want)


def test_short_reads_and_n_seeds(H):
    """a read shorter than o_r + L has no seed in round r, a seed with an N has an empty range: both give range_count 0 and a flag"""
    L, I, max_reseed = 16, 24, 2
    o = ro.reseed_offset(2, I, max_reseed)                  # 16
    assert [v for _, v in ro.seed_positions(o + L - 1, 3, L, I, o)] == [False] * 3
    assert [v for _, v in ro.seed_positions(o + L, 3, L, I, o)] == [True, False, False]
    s, c = ro.range_stats([(5, 9), (1, 0)], [False, True])  # an invalid (short or N) seed, an empty range
    assert (s, c) == (0, 0)
    assert host_flags(H, [s], [c], [300], [1])[0] == 1 and ro.reseed_flag(s, c, 300, True)
    s, c = ro.range_stats([(5, 9), (7, 7), (3, 2)], [True, True, True])
    assert (s, c) == (6, 2)
    assert host_flags(H, [s], [c], [3], [1])[0] == 1 and host_flags(H, [s], [c], [4], [1])[0] == 0
