"""CPU: the per-row {SA, text context} array (nvb_fm_index.ktab_located = 3, nvb_fm_build_rows) changes nothing that
fm_match_locate_one returns.  The host build of the routine (tests/host/rows_harness.cu) runs over the same index and context table
with and without the array -- in one FM_WHOLE call and in the two-pass FM_DEFER / FM_RESUME form of the seed-match stage -- and must give
the same (status, x, y) for every seed: genome-sampled and random seeds, planted exact repeats of whole seeds, k-mers with more than
eight occurrences, tandem repeats, hits at text positions below 16, 4-bit reads with N, and 1 to 17 symbols past the k-mer."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from nvbio_b200.strings import pack_symbols

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "librows_harness.so")
SRC = os.path.join(HERE, "host", "rows_harness.cu")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H():
    deps = [SRC, os.path.join(HERE, "host", "host_harness.cu")] + \
        [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "gotoh_core.cuh", "gotoh_full_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.hr_match_locate.restype = C.c_uint32
    return lib


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


def rows_numpy(full_sa, text):
    """{SA[r], the up to 16 symbols before SA[r], symbol SA[r]-1 lowest} recomputed from the symbols"""
    n = len(text)
    pos = full_sa.astype(np.int64)
    ctx = np.zeros(len(pos), np.uint32)
    live = pos != 0xFFFFFFFF
    for j in range(1, 17):                            # symbol pos - j at bits 2(j-1)
        ok = live & (pos >= j)
        ctx[ok] |= text[pos[ok] - j].astype(np.uint32) << np.uint32(2 * (j - 1))
    assert len(pos) == n + 1
    return np.stack([full_sa.astype(np.uint32), ctx], axis=1).reshape(-1).copy()


def make_index(H, O, text, k):
    n = len(text)
    idx = O.build_index(text)
    full_sa = idx.sa.astype(np.uint32).copy(); full_sa[0] = 0xFFFFFFFF
    gw = pack_symbols(np.concatenate([text, np.zeros(64, np.uint8)]), 2, True)
    ktab = np.zeros(2 * 4 ** k, np.uint32)
    H.hh_fm_build_ktab(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(n), C.c_uint32(idx.primary), C.c_uint32(k), _p(ktab))
    ctx = np.zeros(4 * 4 ** k, np.uint32)
    H.hh_fm_ktab_locate(_p(ktab), _p(full_sa), C.c_uint32(k), _p(ctx))
    H.hh_fm_ktab_context(_p(ctx), C.c_uint32(k), _p(gw), C.c_uint32(n))
    rows = np.zeros(2 * (n + 1), np.uint32)
    H.hr_build_rows(_p(full_sa), _p(gw), C.c_uint32(n), _p(rows))
    return idx, full_sa, gw, ctx, rows


def run(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits, split):
    n = len(full_sa) - 1
    words = np.concatenate([pack_symbols(q, bits, True), np.zeros(4, np.uint32)])
    out = np.zeros((len(offs), 3), np.uint32)
    nd = H.hr_match_locate(_p(idx.bwt_occ), _p(full_sa), _p(idx.L2), C.c_uint32(n), C.c_uint32(idx.primary), _p(gw), _p(words),
                           C.c_uint32(bits), _p(offs), _p(lens), C.c_uint32(len(offs)), _p(ctx), C.c_uint32(k), _p(rows), C.c_int(split), _p(out))
    return out, nd


def seeds(rng, text, k, nq, bits, rem_max=17, plant=()):
    """seeds of k + 1 .. k + rem_max symbols: a third random, the rest from the text (some at position 0..15, some at planted repeats,
    some with one substitution); 4-bit: some with an N"""
    n = len(text)
    lens = (k + rng.integers(1, rem_max + 1, nq)).astype(np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    q = rng.integers(0, 4, int(lens.sum())).astype(np.uint8)
    for i in range(nq):
        L = int(lens[i])
        if i % 3 == 0 or n <= L:
            continue
        if i % 13 == 1:
            st = int(rng.integers(0, min(16, n - L)))                 # hit near the text start
        elif plant and i % 5 == 2:
            st = int(plant[int(rng.integers(0, len(plant)))])         # a planted repeat of the whole seed
        else:
            st = int(rng.integers(0, n - L + 1))
        q[offs[i]:offs[i] + L] = text[st:st + L]
        if i % 7 == 0:
            q[offs[i] + int(rng.integers(0, L))] ^= 1
        if bits == 4 and i % 11 == 0:
            q[offs[i] + int(rng.integers(0, L))] = 4
    return q, offs, lens


def check_same(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits):
    whole_ref, _ = run(H, idx, full_sa, gw, ctx, k, None, q, offs, lens, bits, 0)
    whole, _ = run(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits, 0)
    split_ref, nd_ref = run(H, idx, full_sa, gw, ctx, k, None, q, offs, lens, bits, 1)
    split, nd = run(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits, 1)
    assert np.array_equal(whole, whole_ref)
    assert np.array_equal(split, split_ref)
    assert np.array_equal(split, whole)
    assert nd == nd_ref                                # the first pass's deferral rule does not change
    return whole, nd


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("n,k", [(7250, 6), (116000, 8)])
def test_rows_same_answers(H, O, n, k, bits):
    """n / 4^k ~ 1.77 (bench.py's 1.9 Gbp genome over 15-mers), with planted repeats and a tandem repeat"""
    rng = np.random.default_rng(n + k + bits)
    text = rng.integers(0, 4, n).astype(np.uint8)
    plant = []
    for _ in range(40):                                # exact copies of 30-mers at 2..4 places: seeds that repeat as a whole
        src = int(rng.integers(0, n - 30))
        for _ in range(int(rng.integers(1, 4))):
            dst = int(rng.integers(0, n - 30))
            text[dst:dst + 30] = text[src:src + 30]
        plant.append(src)
    unit = rng.integers(0, 4, 5).astype(np.uint8)     # a tandem repeat: k-mers with far more than eight occurrences
    text[n // 2:n // 2 + 600] = np.tile(unit, 120)
    plant.append(n // 2 + 3)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    assert np.array_equal(rows, rows_numpy(full_sa, text))
    q, offs, lens = seeds(rng, text, k, 6000, bits, plant=plant)
    whole, nd = check_same(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits)
    assert nd > 500 and (whole[:, 0] == 2).sum() > 1000 and (whole[:, 0] == 1).sum() > 50


@pytest.mark.parametrize("bits", [2, 4])
def test_rows_small_texts(H, O, bits):
    """texts shorter than the context, k-mers whose every occurrence lies below position 16, whole-text seeds"""
    rng = np.random.default_rng(11 + bits)
    for n in (5, 17, 40, 90):
        text = rng.integers(0, 2, n).astype(np.uint8)   # a two-letter text: wide ranges on a tiny index
        k = 2
        idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
        assert np.array_equal(rows, rows_numpy(full_sa, text))
        q, offs, lens = seeds(rng, text, k, 400, bits, rem_max=min(17, n))
        check_same(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, bits)


def test_deferred_fraction_scaled_headline(H, O):
    """the premise of the array, on a scaled analogue of bench.py's index (n / 4^k = 1.77: k = 10 over 1.86 Mbp, 20-symbol seeds):
    about half of the genome-sampled seeds and a quarter of the random ones (the read's other strand) land on a k-mer with three or
    more occurrences and are handed to the second pass; the array gives the same answers for all of them"""
    rng = np.random.default_rng(1770)
    k, n, L, nq = 10, int(1.77 * 4 ** 10), 20, 20000
    text = rng.integers(0, 4, n).astype(np.uint8)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    lens = np.full(nq, L, np.uint32)
    offs = (np.arange(nq) * L).astype(np.uint32)
    sampled = np.concatenate([text[s:s + L] for s in rng.integers(0, n - L, nq)]).astype(np.uint8)
    random = rng.integers(0, 4, nq * L).astype(np.uint8)
    fractions = []
    for q in (sampled, random):
        _, nd = check_same(H, idx, full_sa, gw, ctx, k, rows, q, offs, lens, 2)
        fractions.append(nd / nq)
    # Poisson(1.77): P(occurrences >= 3) = 0.53 for a sampled k-mer (one occurrence is its own), 0.26 for a random one
    assert 0.47 < fractions[0] < 0.59 and 0.21 < fractions[1] < 0.31, fractions
