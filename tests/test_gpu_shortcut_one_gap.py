"""-m gpu: the one-gap check of the exact extension shortcut (pipe_perfect_jobs_kernel, gapless_job_shortcut) changes no output.  On a
genome with planted repeats (copies, a homopolymer, period-2 / 3 / 7 tandems) and reads at the headline's error rates plus crafted
ones (two substitutions at chosen spacings, three or four with some at the ends, a 1-2 base indel a few rows from either end, indels and
substitutions inside the tandems, ragged lengths, both strands), nvb_debug_perfect_shortcut 1 (the shortcut with the check), 2 (without
it) and 0 (every job through the DP) give identical outputs: seed_extend's best score, position and hit counts, seed_extend_mapq's
second-best alignment (score, position, strand) and MAPQ, seed_extend_paired's pairs and per-mate MAPQ, and the streaming pipeline."""
import ctypes as C
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import synth
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests.gpu_util import require_gpu
from tests.test_gpu_mapq import packed, outputs, rc
from tests.test_gpu_located_rows import PARAMS, index, best, assert_same

pytestmark = pytest.mark.gpu

N = 400_000
RULES = (1, 2, 0)


def planted_genome(seed=11):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, N).astype(np.uint8)
    a = g[10_000:10_600].copy()
    g[30_000:30_600] = a; g[50_000:50_600] = a                                      # exact copies
    b = a.copy(); b[rng.integers(0, 600, 6)] = rng.integers(0, 4, 6)
    g[70_000:70_600] = b                                                            # a copy with substitutions
    g[90_000:90_600] = rc(a)                                                        # a reverse-complement copy
    for st, period in ((120_000, 1), (140_000, 2), (160_000, 3), (180_000, 7)):
        g[st:st + 2_000] = np.tile(g[st:st + period], 2_000 // period + 1)[:2_000]
    return g


def mutate(r, q, rng):
    r[q] = (r[q] + 1 + rng.integers(0, 3, np.size(q))) % 4


def crafted_reads(g, n_reads, seed, M=150):
    rng = np.random.default_rng(seed)
    reads = []
    spacings = [(p, q) for p in (0, 1, 2, 5, 16, 70, 140, 147) for q in (p + 1, p + 2, p + 9, M - 2, M - 1) if q < M]
    for i in range(n_reads):
        kind = i % 6
        p = int(rng.integers(100, N - 400)) if i % 4 else int(rng.choice([10_000, 30_000, 120_000, 140_000, 160_000, 180_000]) + rng.integers(-100, 1_900))
        m = M if kind != 5 else int(rng.integers(40, M + 1))
        r = g[p:p + m].copy()
        if kind == 0:                                                               # the headline's error rates
            mutate(r, np.flatnonzero(rng.random(m) < 0.01), rng)
        elif kind == 1:                                                             # two substitutions at chosen spacings
            mutate(r, np.array(spacings[i % len(spacings)]), rng)
        elif kind == 2:                                                             # three or four, one at an end
            q = rng.choice(m, int(rng.integers(3, 5)), replace=False); q[0] = rng.integers(0, 3) if i % 2 else m - 1 - rng.integers(0, 3)
            mutate(r, np.unique(q), rng)
        elif kind in (3, 4):                                                        # a 1-2 base indel 1..8 rows from an end
            L = int(rng.integers(1, 3)); k = int(rng.integers(1, 9)); cut = k if i % 2 else m - k
            if kind == 3:
                r = np.concatenate([g[p:p + cut], g[p + cut + L:p + m + L]])
            else:
                r = np.concatenate([g[p:p + cut], rng.integers(0, 4, L).astype(np.uint8), g[p + cut:p + m - L]])
            if rng.integers(0, 2):
                mutate(r, np.array([int(rng.integers(0, m))]), rng)
        else:                                                                       # ragged, 0-2 substitutions
            mutate(r, rng.choice(m, int(rng.integers(0, 3)), replace=False), rng)
        reads.append(rc(r) if rng.integers(0, 2) else r)
    return reads


@pytest.fixture(scope="module")
def setup():
    require_gpu()
    g = planted_genome()
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    return g, gw, index(gw, N, 8)


def each_rule(fn):
    L_ = nb.lib()
    res = []
    try:
        for rule in RULES:
            L_.nvb_debug_perfect_shortcut(C.c_int(rule))
            res.append(fn())
    finally:
        L_.nvb_debug_perfect_shortcut(C.c_int(1))
    for r in res[1:]:
        assert_same(res[0], r, fn.__name__)
    return res[0]


def test_seed_extend_same(setup):
    g, gw, fmi = setup
    params = nb.SeedExtendParams(**PARAMS)
    rs = packed(crafted_reads(g, 12_000, seed=3), L=150)
    L_ = nb.lib()

    def seed_extend():
        return best(nb.seed_extend(fmi, gw, rs, params, hit_capacity=200 * rs.count))
    r = each_rule(seed_extend)
    assert (r["best_score"] > 0).mean() > 0.95
    dp = {}
    try:
        for rule in RULES:                                                          # the check sends clearly fewer jobs to the DP
            L_.nvb_debug_perfect_shortcut(C.c_int(rule))
            ws = nb.seed_extend(fmi, gw, rs, params, hit_capacity=200 * rs.count)
            n = C.c_uint32(0)
            if rule:
                assert L_.nvb_debug_dp_jobs(C.byref(n)) == 0
                dp[rule] = n.value
            del ws
    finally:
        L_.nvb_debug_perfect_shortcut(C.c_int(1))
    assert dp[1] < dp[2]


def test_mapq_same(setup):
    g, gw, fmi = setup
    params = nb.SeedExtendParams(**PARAMS)
    rs = packed(crafted_reads(g, 6_000, seed=5), L=150)

    def mapq():
        ws = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count, mapq=MapqParams.local(150))
        torch.cuda.synchronize()
        return outputs(ws)
    r = each_rule(mapq)
    assert (r["mapq"] < 10).sum() > 50                                              # the repeat families are there


def test_paired_same(setup):
    g, gw, fmi = setup
    n_pairs, L = 4000, 150
    rw, _, _ = synth.sample_pairs(gw, N, n_pairs, L, frag_mean=400, frag_sd=40, sub_rate=0.01, seed=23, mut_seed=24)
    rs = PackedStringSet.fixed(rw.reshape(-1), 2 * n_pairs, L, stride=rw.shape[1] * 16)
    params = nb.SeedExtendParams(**PARAMS)
    pair = nb.PairParams(min_frag=0, max_frag=600, min_mate_score=50)

    def paired():
        ws = nb.seed_extend_paired(fmi, gw, rs, params, pair, hit_capacity=64 * 2 * n_pairs, mapq=MapqParams.local(L))
        torch.cuda.synchronize()
        return {k: getattr(ws, k).cpu().numpy().copy() for k in ("pair_flags", "pair_score", "mate_score", "mate_pos", "mate_strand", "n_rescue",
                                                                 "second_pair_score", "second_mate_pos", "second_mate_strand",
                                                                 "mate_second_score", "mate_mapq")}
    each_rule(paired)


def test_streaming_same(setup):
    g, gw, fmi = setup
    rw, _, _ = synth.sample_reads(gw, N, 4000, 150, seed=33, mut_seed=34)
    host = rw.cpu().pin_memory()

    def streaming():
        st = nb.StreamingSeedExtend(fmi, gw, nb.SeedExtendParams(), 4000, 150, rw.shape[1], hit_capacity=256000, depth=2)
        try:
            t = st.submit(host)
            return {str(j): v.cpu().numpy() for j, v in enumerate(st.result(t))}
        finally:
            st.close()
    each_rule(streaming)
