"""CPU: the wide k-mer table (32-byte entries, nvb_fm_index.ktab_located = 4 / 5, nvb_fm_build_ktab_wide) changes nothing that
fm_match_locate_one or fm_match_one returns.  The host build (tests/host/wide_harness.cu) fills the table with the builder's own
per-entry routine, which is checked entry by entry against a numpy restatement; then every seed gets the same (status, x, y) over the
same index with the 16-byte context table (levels 2 / 3) and with the wide one (levels 4 / 5), in one FM_WHOLE call and in the
FM_DEFER / FM_RESUME form, with and without the per-row array.  Seeds: genome-sampled and random, planted whole-seed repeats, tandem
repeats, hits below text position 16, tiny texts, 4-bit reads with N, 1 to 17 symbols past the k-mer."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from tests.test_located_rows import make_index, seeds, _p

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "libwide_harness.so")
SRC = os.path.join(HERE, "host", "wide_harness.cu")


@pytest.fixture(scope="module")
def H():
    deps = [SRC, os.path.join(HERE, "host", "rows_harness.cu"), os.path.join(HERE, "host", "host_harness.cu")] + \
        [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "gotoh_core.cuh", "gotoh_full_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.hw_match_locate.restype = C.c_uint32
    return lib


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


def aligned_u32(n_words, align=32):
    """a zeroed uint32 array whose data is `align`-byte aligned (the wide table's requirement)"""
    raw = np.zeros(n_words + align // 4, np.uint32)
    skip = (-raw.ctypes.data % align) // 4
    return raw[skip:skip + n_words]


def ktab8_of(H, idx, n, k):
    t = np.zeros(2 * 4 ** k, np.uint32)
    H.hh_fm_build_ktab(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(n), C.c_uint32(idx.primary), C.c_uint32(k), _p(t))
    return t


def build_wide(H, ktab8, full_sa, gw, n, k):
    w = aligned_u32(8 * 4 ** k)
    H.hw_build_wide(_p(ktab8), _p(full_sa), _p(gw), C.c_uint32(n), C.c_uint32(k), _p(w))
    return w


def wide_numpy(ktab8, full_sa, text):
    """the 32-byte entries recomputed from the ranges, the suffix array and the symbols"""
    n = len(text)
    x = ktab8[0::2].astype(np.int64); y = ktab8[1::2].astype(np.int64)
    w = np.zeros((len(x), 8), np.uint32)
    w[:, 0] = x; w[:, 1] = y
    d = np.where(x <= y, y - x, -1)

    def ctx(pos, want):
        out = np.zeros(len(pos), np.uint32)
        live = pos != 0xFFFFFFFF
        for j in range(1, want + 1):
            ok = live & (pos >= j)
            out[ok] |= text[pos[ok] - j].astype(np.uint32) << np.uint32(2 * (j - 1))
        return out

    def sa(sel, i):
        return full_sa[x[sel] + i].astype(np.int64)

    s = d == 0
    w[s, 2] = sa(s, 0); w[s, 3] = ctx(sa(s, 0), 16)
    s = d == 1
    w[s, 2] = sa(s, 0); w[s, 3] = sa(s, 1)
    assert n < 0xC0000000
    w[s, 1] = 0xC0000000 | ctx(sa(s, 0), 7) | (ctx(sa(s, 1), 7) << np.uint32(14))
    s = d == 2
    for i in range(3):
        w[s, 2 + i] = sa(s, i); w[s, 5 + i] = ctx(sa(s, i), 16)
    for dd in range(3, 8):
        s = d == dd
        for i in range(dd + 1):
            w[s, 2 + i // 2] |= ctx(sa(s, i), 8) << np.uint32(16 * (i & 1))
            if dd == 3:
                w[s, 4 + i] = sa(s, i)
    return w.reshape(-1)


def run(H, idx, full_sa, gw, tab, k, level, rows, q, offs, lens, bits, split):
    n = len(full_sa) - 1
    words = np.concatenate([pack(q, bits), np.zeros(4, np.uint32)])
    out = np.zeros((len(offs), 3), np.uint32)
    nd = H.hw_match_locate(_p(idx.bwt_occ), _p(full_sa), _p(idx.L2), C.c_uint32(n), C.c_uint32(idx.primary), _p(gw), _p(words),
                           C.c_uint32(bits), _p(offs), _p(lens), C.c_uint32(len(offs)), _p(tab), C.c_uint32(k), C.c_uint32(level),
                           _p(rows), C.c_int(split), _p(out))
    return out, nd


def pack(q, bits):
    from nvbio_b200.strings import pack_symbols
    return pack_symbols(q, bits, True)


def check_same(H, idx, full_sa, gw, ctx, wide, k, rows, q, offs, lens, bits):
    """every seed: the same (status, x, y) at levels 2, 3, 4, 5, one call and two passes; returns the level-2 result and the number
    of seeds the first pass hands on at level 2 and at level 4"""
    ref, nd_ref = run(H, idx, full_sa, gw, ctx, k, 2, None, q, offs, lens, bits, 0)
    nds = {}
    for level, tab, rw in ((2, ctx, None), (3, ctx, rows), (4, wide, None), (5, wide, rows)):
        for split in (0, 1):
            out, nd = run(H, idx, full_sa, gw, tab, k, level, rw, q, offs, lens, bits, split)
            assert np.array_equal(out, ref), (level, split, np.flatnonzero((out != ref).any(axis=1))[:10])
            if split:
                nds[level] = nd
    assert nds[3] == nds[2] and nds[5] == nds[4] and nds[4] <= nds[2]
    return ref, nds[2], nds[4]


def planted_text(rng, n, k):
    text = rng.integers(0, 4, n).astype(np.uint8)
    plant = []
    for _ in range(60):                                # exact copies of 30-mers at 2..4 places: seeds that repeat as a whole
        src = int(rng.integers(0, n - 30))
        for _ in range(int(rng.integers(1, 4))):
            dst = int(rng.integers(0, n - 30))
            text[dst:dst + 30] = text[src:src + 30]
        plant.append(src)
    unit = rng.integers(0, 4, 5).astype(np.uint8)     # a tandem repeat: k-mers with far more than eight occurrences
    text[n // 2:n // 2 + 600] = np.tile(unit, 120)
    plant.append(n // 2 + 3)
    return text, plant


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("n,k", [(7250, 6), (116000, 8)])
def test_wide_same_answers(H, O, n, k, bits):
    """n / 4^k ~ 1.77 (bench.py's 1.9 Gbp genome over 15-mers), with planted repeats and a tandem repeat; the seeds cover k-mers with
    3, 4 and 5-8 occurrences with no survivor, one located survivor, one survivor isolated by the last step and a whole-seed repeat,
    and k-mers with more than eight"""
    rng = np.random.default_rng(n + k + bits + 1)
    text, plant = planted_text(rng, n, k)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    k8 = ktab8_of(H, idx, n, k)
    wide = build_wide(H, k8, full_sa, gw, n, k)
    assert np.array_equal(wide, wide_numpy(k8, full_sa, text))
    # the first 16 bytes are the level-2 entry, except where level 2 leaves words 2-3 of a 3..8-row entry zero
    w4 = wide.reshape(-1, 8)[:, :4]; c4 = ctx.reshape(-1, 4)
    d = k8[1::2].astype(np.int64) - k8[0::2].astype(np.int64)
    keep = ~((d >= 2) & (d <= 7))
    assert np.array_equal(w4[keep], c4[keep]) and np.array_equal(w4[~keep, :2], c4[~keep, :2]) and not c4[~keep, 2:].any()
    q, offs, lens = seeds(rng, text, k, 8000, bits, plant=plant)
    ref, nd2, nd4 = check_same(H, idx, full_sa, gw, ctx, wide, k, rows, q, offs, lens, bits)
    assert nd4 < nd2
    # coverage: the k-mer's number of rows (from the table) against the walk's answer
    sym = np.array([q[o + L - k:o + L] for o, L in zip(offs, lens)])
    has_n = (sym > 3).any(axis=1)
    u = np.zeros(len(offs), np.int64)
    for j in range(k):
        u = u * 4 + (sym[:, j] & 3)
    nr = np.where(has_n, 0, d[u] + 1)
    st, x, y = ref[:, 0], ref[:, 1].astype(np.int64), ref[:, 2].astype(np.int64)
    kinds = {"empty": st == 0, "located": st == 2, "last_step": (st == 1) & (x == y), "repeat": (st == 1) & (y > x)}
    for lo, hi in ((3, 3), (4, 4), (5, 8)):
        cls = (nr >= lo) & (nr <= hi)
        for name, m in kinds.items():
            assert (cls & m).any(), (lo, hi, name)
    assert (nr >= 9).sum() > 50


@pytest.mark.parametrize("bits", [2, 4])
def test_wide_small_texts(H, O, bits):
    """texts shorter than the context, k-mers whose every occurrence lies below position 16, whole-text seeds"""
    rng = np.random.default_rng(21 + bits)
    for n in (5, 17, 40, 90):
        text = rng.integers(0, 2, n).astype(np.uint8)   # a two-letter text: wide ranges on a tiny index
        k = 2
        idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
        k8 = ktab8_of(H, idx, n, k)
        wide = build_wide(H, k8, full_sa, gw, n, k)
        assert np.array_equal(wide, wide_numpy(k8, full_sa, text))
        q, offs, lens = seeds(rng, text, k, 400, bits, rem_max=min(17, n))
        check_same(H, idx, full_sa, gw, ctx, wide, k, rows, q, offs, lens, bits)


@pytest.mark.parametrize("bits", [2, 4])
def test_wide_match_ranges(H, O, bits):
    """fm_match_one (nvb_fm_match's routine) reads only the range of an entry: the same ranges from the 8-byte, 16-byte and 32-byte
    tables, in every consumption order"""
    rng = np.random.default_rng(31 + bits)
    n, k = 20000, 7
    text, plant = planted_text(rng, n, k)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    k8 = ktab8_of(H, idx, n, k)
    wide = build_wide(H, k8, full_sa, gw, n, k)
    q, offs, lens = seeds(rng, text, k, 3000, bits, plant=plant)
    words = np.concatenate([pack(q, bits), np.zeros(4, np.uint32)])
    for flags in (0, 1, 2, 3):
        outs = []
        for level, tab in ((0, k8), (2, ctx), (4, wide)):
            out = np.zeros(2 * len(offs), np.uint32)
            H.hw_match(_p(idx.bwt_occ), _p(full_sa), _p(idx.L2), C.c_uint32(n), C.c_uint32(idx.primary), _p(words), C.c_uint32(bits),
                       _p(offs), _p(lens), C.c_uint32(len(offs)), C.c_uint32(flags), _p(tab), C.c_uint32(k), C.c_uint32(level), _p(out))
            outs.append(out)
        assert np.array_equal(outs[1], outs[0]) and np.array_equal(outs[2], outs[0]), flags


def test_deferred_fraction_scaled_headline(H, O):
    """the premise of the wide table, on a scaled analogue of bench.py's index and seeds (n / 4^k = 1.77: k = 10 over 1.86 Mbp,
    seeds of k + 5 symbols): with the 16-byte table the first pass hands on about half of the genome-sampled seeds and a quarter of the
    random ones (the read's other strand); with the wide one about a tenth and almost none, and every answer is the same"""
    rng = np.random.default_rng(1771)
    k, L, nq = 10, 15, 20000
    n = int(1.77 * 4 ** k)
    text = rng.integers(0, 4, n).astype(np.uint8)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    k8 = ktab8_of(H, idx, n, k)
    wide = build_wide(H, k8, full_sa, gw, n, k)
    lens = np.full(nq, L, np.uint32)
    offs = (np.arange(nq) * L).astype(np.uint32)
    sampled = np.concatenate([text[s:s + L] for s in rng.integers(0, n - L, nq)]).astype(np.uint8)
    random = rng.integers(0, 4, nq * L).astype(np.uint8)
    before, after = [], []
    for q in (sampled, random):
        _, nd2, nd4 = check_same(H, idx, full_sa, gw, ctx, wide, k, rows, q, offs, lens, 2)
        before.append(nd2 / nq); after.append(nd4 / nq)
    assert 0.45 < before[0] < 0.57 and 0.21 < before[1] < 0.31, before
    assert after[0] < 0.13 and after[1] < 0.01 and sum(after) / 2 < 0.06, after
