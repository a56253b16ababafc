"""-m gpu: the per-row {SA, text context} array (FMIndexDevice.rows, nvb_fm_build_rows) built on the device equals its host
recomputation, and the same index with the array present and detached gives identical outputs on every path that resolves seeds:
seed_extend on the per-read path (one- and two-pass seed match), seed_extend_mapq, seed_extend_paired and the streaming pipeline,
for 2-bit reads and 4-bit reads with N, on a random genome with n / 4^k ~ 1.77 and on a repeat-rich one."""
import ctypes as C
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet, pack_symbols, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.test_gpu_mapq import repeat_genome, make_reads, packed, outputs, N_GENOME
from tests.test_located_rows import rows_numpy

pytestmark = pytest.mark.gpu

PARAMS = dict(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
              scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


def index(gw, n, k):
    fmi, _ = nb.FMIndexDevice.from_text(gw, n, sa_interval=1)
    fmi.build_ktab(k, located=True, text=gw)
    assert fmi.rows is not None and fmi.ktab_located == 2 and fmi.struct().ktab_located == 3
    return fmi


@pytest.fixture(scope="module")
def random_setup():
    require_gpu()
    k = 9
    n = int(1.77 * 4 ** k)
    gw = synth.random_genome_words(n, seed=177)
    return gw, n, index(gw, n, k)


@pytest.fixture(scope="module")
def repeat_setup():
    require_gpu()
    g = repeat_genome(seed=8)
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    return g, gw, index(gw, N_GENOME, 8)


def with_and_without(fmi, fn):
    """fn() with the array, then with it detached; returns both results"""
    rows = fmi.rows
    a = fn()
    fmi.rows = None
    try:
        b = fn()
    finally:
        fmi.rows = rows
    return a, b


def best(ws):
    torch.cuda.synchronize()
    return dict(best_score=ws.best_score.cpu().numpy(), best_pos=host_u32(ws.best_pos).copy(), n_hits=ws.n_hits.cpu().numpy())


def assert_same(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k]), (what, k)


def test_rows_equal_host_recomputation(random_setup):
    gw, n, fmi = random_setup
    text = unpack_symbols(host_u32(gw), n)
    assert fmi.rows.shape == (n + 1, 2)
    assert np.array_equal(host_u32(fmi.rows).reshape(-1), rows_numpy(host_u32(fmi.ssa), text))
    assert fmi.nbytes() == fmi.bwt_occ.numel() * 4 + fmi.ssa.numel() * 4 + fmi.ktab.numel() * 4 + (n + 1) * 8


@pytest.mark.parametrize("split", [1, 0])
def test_seed_extend_same(random_setup, repeat_setup, split):
    """per-read path, two-pass (split = 1) and one-pass seed match, 2-bit reads from bench's sampler and 4-bit reads with N"""
    L_ = nb.lib()
    gw, n, fmi = random_setup
    params = nb.SeedExtendParams(**PARAMS)
    rw, _, _ = synth.sample_reads(gw, n, 20000, 150, sub_rate=0.01, indel_rate=0.001, seed=5, mut_seed=6)
    rs = PackedStringSet.fixed(rw.reshape(-1), 20000, 150, stride=rw.shape[1] * 16)
    g, gw2, fmi2 = repeat_setup
    reads = make_reads(g, n_reads=4000, seed=17)
    rng = np.random.default_rng(4)
    for r in reads[::5]:
        r[rng.integers(0, len(r), 2)] = 4
    rs4 = packed(reads, 4)
    L_.nvb_debug_seed_split(C.c_int(split))
    try:
        for f, genome, reads_set, what in ((fmi, gw, rs, "random, 2-bit"), (fmi2, gw2, rs4, "repeats, 4-bit"), (fmi2, gw2, packed(reads, 2), "repeats, 2-bit")):
            a, b = with_and_without(f, lambda: best(nb.seed_extend(f, genome, reads_set, params, hit_capacity=200 * reads_set.count)))
            assert_same(a, b, what)
            assert int(a["n_hits"][0]) == int(a["n_hits"][1])
    finally:
        L_.nvb_debug_seed_split(C.c_int(1))


def test_mapq_same(repeat_setup):
    g, gw, fmi = repeat_setup
    reads = make_reads(g, n_reads=3000, ragged=True, seed=29)
    rs = packed(reads)
    params = nb.SeedExtendParams(**PARAMS)
    mq = MapqParams.local(100)

    def run():
        ws = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count, mapq=mq)
        torch.cuda.synchronize()
        return outputs(ws)
    a, b = with_and_without(fmi, run)
    assert_same(a, b, "mapq")
    assert (a["mapq"] < 10).sum() > 100                       # the repeat families are there


def test_paired_same(random_setup):
    gw, n, fmi = random_setup
    n_pairs, L = 3000, 100
    rw, _, _ = synth.sample_pairs(gw, n, n_pairs, L, frag_mean=300, frag_sd=40, sub_rate=0.02, hard_frac=0.3, hard_sub_rate=0.2, seed=21, mut_seed=22)
    rs = PackedStringSet.fixed(rw.reshape(-1), 2 * n_pairs, L, stride=rw.shape[1] * 16)
    params = nb.SeedExtendParams(**PARAMS)
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)

    def run():
        ws = nb.seed_extend_paired(fmi, gw, rs, params, pair, hit_capacity=64 * 2 * n_pairs)
        torch.cuda.synchronize()
        return {k: getattr(ws, k).cpu().numpy().copy() for k in ("pair_flags", "pair_score", "mate_score", "mate_pos", "mate_strand", "n_rescue")}
    a, b = with_and_without(fmi, run)
    assert_same(a, b, "paired")


def test_streaming_same(random_setup):
    gw, n, fmi = random_setup
    rw, _, _ = synth.sample_reads(gw, n, 2000, 150, seed=31, mut_seed=32)
    host = rw.cpu().pin_memory()

    def run():
        st = nb.StreamingSeedExtend(fmi, gw, nb.SeedExtendParams(), 2000, 150, rw.shape[1], hit_capacity=128000, depth=2)
        try:
            t = st.submit(host)
            return [v.clone() for v in st.result(t)]
        finally:
            st.close()
    a, b = with_and_without(fmi, run)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
