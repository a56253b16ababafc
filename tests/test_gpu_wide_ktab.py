"""-m gpu: the wide k-mer table (32-byte entries, nvb_fm_build_ktab_wide) built on the device equals its host restatement,
build_ktab picks it exactly when a 16-byte table would not fit the L2 cache, and a second index over the same arrays with the wide table
gives outputs identical to the 16-byte one on every path that resolves seeds: seed_extend on the per-read path (one- and two-pass seed
match), seed_extend_mapq, seed_extend_paired, the streaming pipeline and nb.match ranges -- with and without the per-row array, for
2-bit reads and 4-bit reads with N, on a random genome with n / 4^k ~ 1.77 and on a repeat-rich one."""
import ctypes as C
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import synth
from nvbio_b200._lib import lib, check
from nvbio_b200.fmindex import match, _stream
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet, pack_symbols, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.test_gpu_mapq import repeat_genome, make_reads, packed, outputs, N_GENOME
from tests.test_gpu_located_rows import PARAMS, index, best, assert_same
from tests.test_wide_ktab import wide_numpy

pytestmark = pytest.mark.gpu


def wide_twin(fmi, gw):
    """a second index over fmi's arrays (and its per-row array) with the wide table of the same k, built through the C entry point"""
    w = nb.FMIndexDevice(fmi.bwt_occ, fmi.ssa, fmi.L2, fmi.length, fmi.primary, sa_interval=1)
    tab = torch.empty((4 ** fmi.ktab_k, 8), dtype=torch.int32, device=fmi.device)
    assert tab.data_ptr() % 32 == 0
    check(lib().nvb_fm_build_ktab_wide(C.byref(w.struct()), C.c_uint32(fmi.ktab_k), C.c_void_p(gw.data_ptr()), C.c_void_p(tab.data_ptr()),
                                       _stream()), "nvb_fm_build_ktab_wide")
    w.ktab, w.ktab_k, w.ktab_located, w.ktab_wide, w.rows = tab, fmi.ktab_k, 2, True, fmi.rows
    assert w.struct().ktab_located == 5
    return w


@pytest.fixture(scope="module")
def random_setup():
    require_gpu()
    k = 9
    n = int(1.77 * 4 ** k)
    gw = synth.random_genome_words(n, seed=178)
    fmi = index(gw, n, k)
    return gw, n, fmi, wide_twin(fmi, gw)


@pytest.fixture(scope="module")
def repeat_setup():
    require_gpu()
    g = repeat_genome(seed=9)
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    fmi = index(gw, N_GENOME, 8)
    return g, gw, fmi, wide_twin(fmi, gw)


def variants(fmi, wide, fn):
    """fn(index) on the 16-byte table with the per-row array, the wide table with it and the wide table without it"""
    rows = wide.rows
    a, b = fn(fmi), fn(wide)
    wide.rows = None
    try:
        c = fn(wide)
    finally:
        wide.rows = rows
    return a, b, c


def all_same(res, what):
    for r in res[1:]:
        assert_same(res[0], r, what)


def test_wide_table_equals_host_restatement(random_setup, repeat_setup):
    for gw, n, fmi, wide in (random_setup, repeat_setup[1:2] + (N_GENOME,) + repeat_setup[2:]):
        text = unpack_symbols(host_u32(gw), n)
        ctx = host_u32(fmi.ktab).reshape(-1, 4)
        x, y = ctx[:, 0].copy(), ctx[:, 1].copy()
        two = y >= 0xC0000000
        y[two] = x[two] + 1
        k8 = np.stack([x, y], axis=1).reshape(-1)
        assert np.array_equal(host_u32(wide.ktab).reshape(-1), wide_numpy(k8, host_u32(fmi.ssa), text))
        assert wide.nbytes() == fmi.nbytes() + fmi.ktab.numel() * 4          # twice the table, the same rest


def test_build_ktab_picks_wide_above_l2():
    require_gpu()
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    k = 2
    while 4 ** k * 16 <= l2:
        k += 1
    n = 200_000
    gw = synth.random_genome_words(n, seed=5)
    fmi, _ = nb.FMIndexDevice.from_text(gw, n, sa_interval=1)
    fmi.build_ktab(k - 1, located=True, text=gw)
    assert not fmi.ktab_wide and fmi.struct().ktab_located == 3 and fmi.ktab.shape == (4 ** (k - 1), 4)
    fmi.build_ktab(k, located=True, text=gw)
    assert fmi.ktab_wide and fmi.ktab_located == 2 and fmi.struct().ktab_located == 5 and fmi.ktab.shape == (4 ** k, 8)
    assert fmi.nbytes() == fmi.bwt_occ.numel() * 4 + fmi.ssa.numel() * 4 + 4 ** k * 32 + (n + 1) * 8
    rw, _, _ = synth.sample_reads(gw, n, 3000, 150, sub_rate=0.01, seed=7, mut_seed=8)
    rs = PackedStringSet.fixed(rw.reshape(-1), 3000, 150, stride=rw.shape[1] * 16)
    params = nb.SeedExtendParams(**PARAMS)
    a = best(nb.seed_extend(fmi, gw, rs, params, hit_capacity=200 * rs.count))
    fmi.build_ktab(k, located=True)                                          # no text: the 16-byte located table
    assert not fmi.ktab_wide and fmi.struct().ktab_located == 1
    b = best(nb.seed_extend(fmi, gw, rs, params, hit_capacity=200 * rs.count))
    assert_same(a, b, "k above the L2 size")


@pytest.mark.parametrize("split", [1, 0])
def test_seed_extend_same(random_setup, repeat_setup, split):
    """per-read path, two-pass (split = 1) and one-pass seed match, 2-bit reads from bench's sampler and 4-bit reads with N"""
    L_ = nb.lib()
    gw, n, fmi, wide = random_setup
    params = nb.SeedExtendParams(**PARAMS)
    rw, _, _ = synth.sample_reads(gw, n, 20000, 150, sub_rate=0.01, indel_rate=0.001, seed=15, mut_seed=16)
    rs = PackedStringSet.fixed(rw.reshape(-1), 20000, 150, stride=rw.shape[1] * 16)
    g, gw2, fmi2, wide2 = repeat_setup
    reads = make_reads(g, n_reads=4000, seed=18)
    rng = np.random.default_rng(5)
    for r in reads[::5]:
        r[rng.integers(0, len(r), 2)] = 4
    L_.nvb_debug_seed_split(C.c_int(split))
    try:
        for f, w, genome, reads_set, what in ((fmi, wide, gw, rs, "random, 2-bit"), (fmi2, wide2, gw2, packed(reads, 4), "repeats, 4-bit"),
                                              (fmi2, wide2, gw2, packed(reads, 2), "repeats, 2-bit")):
            res = variants(f, w, lambda i: best(nb.seed_extend(i, genome, reads_set, params, hit_capacity=200 * reads_set.count)))
            all_same(res, what)
    finally:
        L_.nvb_debug_seed_split(C.c_int(1))


def test_mapq_same(repeat_setup):
    g, gw, fmi, wide = repeat_setup
    rs = packed(make_reads(g, n_reads=3000, ragged=True, seed=30))
    params = nb.SeedExtendParams(**PARAMS)
    mq = MapqParams.local(100)

    def run(i):
        ws = nb.seed_extend(i, gw, rs, params, hit_capacity=1000 * rs.count, mapq=mq)
        torch.cuda.synchronize()
        return outputs(ws)
    res = variants(fmi, wide, run)
    all_same(res, "mapq")
    assert (res[0]["mapq"] < 10).sum() > 100                  # the repeat families are there


@pytest.mark.parametrize("which", ["random", "repeats"])
def test_paired_same(random_setup, repeat_setup, which):
    gw, n, fmi, wide = random_setup if which == "random" else (repeat_setup[1], N_GENOME, repeat_setup[2], repeat_setup[3])
    n_pairs, L = 3000, 100
    rw, _, _ = synth.sample_pairs(gw, n, n_pairs, L, frag_mean=300, frag_sd=40, sub_rate=0.02, hard_frac=0.3, hard_sub_rate=0.2, seed=23, mut_seed=24)
    rs = PackedStringSet.fixed(rw.reshape(-1), 2 * n_pairs, L, stride=rw.shape[1] * 16)
    params = nb.SeedExtendParams(**PARAMS)
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)

    def run(i):
        ws = nb.seed_extend_paired(i, gw, rs, params, pair, hit_capacity=64 * 2 * n_pairs)
        torch.cuda.synchronize()
        return {k: getattr(ws, k).cpu().numpy().copy() for k in ("pair_flags", "pair_score", "mate_score", "mate_pos", "mate_strand", "n_rescue")}
    all_same(variants(fmi, wide, run), "paired " + which)


def test_streaming_same(random_setup):
    gw, n, fmi, wide = random_setup
    rw, _, _ = synth.sample_reads(gw, n, 2000, 150, seed=33, mut_seed=34)
    host = rw.cpu().pin_memory()

    def run(i):
        st = nb.StreamingSeedExtend(i, gw, nb.SeedExtendParams(), 2000, 150, rw.shape[1], hit_capacity=128000, depth=2)
        try:
            t = st.submit(host)
            return {str(j): v.cpu().numpy() for j, v in enumerate(st.result(t))}
        finally:
            st.close()
    all_same(variants(fmi, wide, run), "streaming")


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_match_ranges_same(random_setup, repeat_setup, flags):
    for gw, n, fmi, wide in (random_setup, (repeat_setup[1], N_GENOME, repeat_setup[2], repeat_setup[3])):
        rw, _, _ = synth.sample_reads(gw, n, 5000, 24, sub_rate=0.02, seed=41, mut_seed=42)
        qs = PackedStringSet.fixed(rw.reshape(-1), 5000, 24, stride=rw.shape[1] * 16)
        a, b = match(fmi, qs, flags), match(wide, qs, flags)
        assert torch.equal(a, b), flags
