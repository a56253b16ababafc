"""-m gpu: second-best pair and paired MAPQ of nvb_seed_extend_paired_mapq against the oracle composition (tests/pair_mapq_oracle.py) on a
genome with planted repeat families, the same outputs on every code path, the pair outputs of nvb_seed_extend_paired, and the single-end
MAPQ of nvb_seed_extend_mapq for the mates of unpaired pairs."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import pack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.test_gpu_mapq import rc, packed
from tests.pair_mapq_oracle import pair_mapq_oracle, INT_MIN

pytestmark = pytest.mark.gpu

N_GENOME = 200_000
L = 100
PAIR_OUTPUTS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand")
MAPQ_OUTPUTS = ("second_pair_score", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")
REPEAT_UNIT = (100_000, 120)                                 # copied four times: a mate inside it is a repeat, its partner is unique


def pair_genome(seed=11):
    """random genome with, for 100 bp mates and fragments up to 400: a 1000 bp segment copied exactly (longer than any fragment), a
    family of 800 bp copies with 1, 2 and 3 substitutions per 100 bp, a 120 bp unit copied four times far apart, a reverse-complement
    copy, period-40 and period-52 tandems (below / above len/2) and a 150 bp unit copied 200 times, 230 bp apart"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, N_GENOME).astype(np.uint8)
    g[40_000:41_000] = g[20_000:21_000]
    b = g[60_000:60_800].copy()
    for start, step in ((70_000, 100), (76_000, 50), (82_000, 33)):
        c = b.copy(); c[step // 2::step] = (c[step // 2::step] + 1) % 4
        g[start:start + 800] = c
    st, ln = REPEAT_UNIT
    for at in (130_000, 135_000, 140_000, 145_000):
        g[at:at + ln] = g[st:st + ln]
    g[95_000:95_400] = rc(g[90_000:90_400])
    g[110_000:110_800] = np.tile(g[110_000:110_040], 20)
    g[120_000:120_832] = np.tile(g[120_000:120_052], 16)
    unit = g[150_000:150_150].copy()
    for k in range(200):
        g[150_000 + 230 * k:150_000 + 230 * k + 150] = unit
    return g


REGIONS = {0: (20_000, 1000), 1: (60_000, 800), 3: (110_000, 800), 4: (90_000, 400), 5: (150_000, 46_000)}


def make_pairs(g, n_pairs=1000, ragged=False, seed=3):
    """mate 1 of every pair, then mate 2; kind[p] = p % 10: 0 exact 1000 bp copy, 1 substitution family, 2 one mate inside the four-copy
    unit (repeat_mate[p] says which), 3 tandems, 4 reverse-complement copy, 5 the 200-copy unit, 6 unique, 7 unique with mate 2 heavily
    mutated (rescues), 8 unpaired (fragment of 2000) or mate 2 unaligned (random), 9 unique with substitutions"""
    rng = np.random.default_rng(seed)
    m1s, m2s, repeat_mate = [], [], np.full(n_pairs, -1)
    for p in range(n_pairs):
        kind = p % 10
        l1, l2 = (int(rng.integers(L - 40, L + 1)) if ragged else L for _ in range(2))
        if kind == 3:
            st, span = (110_000, 800) if rng.random() < 0.5 else (120_000, 832)
        else:
            st, span = REGIONS.get(kind, (0, 140_000))
        f = int(rng.integers(max(l1, l2) + 20, 381))
        if kind == 2:
            left = REPEAT_UNIT[0] + int(rng.integers(0, REPEAT_UNIT[1] - l1 + 1))
        elif kind == 8 and p % 20 == 8:
            left, f = int(rng.integers(0, 130_000)), 2000
        else:
            left = st + int(rng.integers(0, max(span - f, 0) + 1))
        a = g[left:left + l1].copy()
        b = rc(g[left + f - l2:left + f])
        if kind == 7:
            m = rng.random(l2) < 0.12
            b[m] = (b[m] + 1) % 4
        elif kind == 8 and p % 20 == 18:
            b = rng.integers(0, 4, l2).astype(np.uint8)
        elif kind == 9:
            a[rng.integers(0, l1, 2)] = rng.integers(0, 4, 2); b[rng.integers(0, l2, 2)] = rng.integers(0, 4, 2)
        swap = rng.random() < 0.5
        if kind == 2:
            repeat_mate[p] = 1 if swap else 0
        m1s.append(b if swap else a); m2s.append(a if swap else b)
    return m1s + m2s, repeat_mate


@pytest.fixture(scope="module")
def setup():
    require_gpu()
    O = orc.Oracle()
    g = pair_genome()
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    return O, g, gw, idx, fmi


def se_params(**kw):
    a = dict(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    a.update(kw)
    return nb.SeedExtendParams(**a)


def run(fmi, gw, rs, params, pair, mq=None):
    ws = nb.seed_extend_paired(fmi, gw, rs, params, pair, hit_capacity=1000 * rs.count, mapq=mq)
    torch.cuda.synchronize()
    return ws


def outputs(ws, mapq=True):
    out = {}
    for k in PAIR_OUTPUTS + (MAPQ_OUTPUTS if mapq else ()) + ("n_rescue", "n_hits"):
        t = getattr(ws, k)
        out[k] = host_u32(t).astype(np.int64) if k in ("mate_pos", "second_mate_pos") else t.cpu().numpy().astype(np.int64)
    return out


def check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, pair, mq, quals=None):
    n = len(reads) // 2
    ws = run(fmi, gw, rs, params, pair, mq)
    got = outputs(ws)
    assert got["n_hits"][0] == got["n_hits"][1]                                    # no hit dropped: the oracle keeps them all
    want = pair_mapq_oracle(O, idx, g, reads, params, pair, n, mq.min_score.cpu().numpy(), mq.match_bonus, quals=quals)
    assert tuple(got["n_rescue"]) == tuple(want["n_rescue"])
    for k in PAIR_OUTPUTS + MAPQ_OUTPUTS:
        bad = np.argwhere(got[k] != want[k])
        assert len(bad) == 0, (k, [(tuple(int(v) for v in i), int(got[k][tuple(i)]), int(want[k][tuple(i)])) for i in bad[:5]])
    # the pair outputs are nvb_seed_extend_paired's
    plain = outputs(run(fmi, gw, rs, params, pair), mapq=False)
    for k in PAIR_OUTPUTS + ("n_rescue", "n_hits"):
        assert np.array_equal(plain[k], got[k]), k
    # the mates of unpaired pairs get nvb_seed_extend_mapq's single-end outputs on the same 2n reads; every mate its second score
    se = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count, mapq=mq)
    torch.cuda.synchronize()
    un = got["pair_flags"] == nb.pipeline.PAIR_UNPAIRED
    se_mapq = se.mapq.cpu().numpy().astype(np.int64).reshape(2, n)
    assert np.array_equal(got["mate_mapq"][:, un], se_mapq[:, un])
    assert np.array_equal(got["mate_second_score"].reshape(-1), se.second_score.cpu().numpy())
    # the outputs cover the interesting cases
    flags = got["pair_flags"]
    has2 = got["second_pair_score"] != INT_MIN
    assert (flags == 1).sum() > 0.4 * n and ((flags == 2) | (flags == 4)).sum() > 5 and un.sum() > 10
    assert (got["mate_score"] == INT_MIN).sum() > 5 and (got["mate_mapq"][got["mate_score"] == INT_MIN] == 0).all()
    assert has2[flags != 0].sum() > 0.1 * n and (~has2[flags != 0]).sum() > 0.2 * n
    assert (has2 & (got["second_pair_score"] == got["pair_score"])).sum() > 20
    assert (got["second_mate_pos"][:, ~has2] == 0xFFFFFFFF).all() and (got["second_mate_strand"][:, ~has2] == 0).all()
    assert (got["mate_mapq"][0, flags != 0] == got["mate_mapq"][1, flags != 0]).all()
    return got, se_mapq


@pytest.mark.parametrize("bits,ragged", [(2, False), (4, True)])
def test_paired_mapq_vs_oracle(setup, bits, ragged):
    O, g, gw, idx, fmi = setup
    reads, repeat_mate = make_pairs(g, ragged=ragged, seed=3 + bits)
    if bits == 4:
        rng = np.random.default_rng(5)
        for r in reads[::9]:
            r[rng.integers(0, len(r), 2)] = 4                                        # N
    rs = packed(reads, bits)
    pair = nb.PairParams(min_frag=0, max_frag=400, min_mate_score=60)
    got, se_mapq = check_vs_oracle(O, g, idx, fmi, gw, reads, rs, se_params(), pair, MapqParams.local(L))
    if bits == 2:
        n = len(reads) // 2
        kind = np.arange(n) % 10
        conc = got["pair_flags"] == 1
        # a pair inside the exact 1000 bp copy has an equally good distinct pair: MAPQ 0 or 1
        sel = (kind == 0) & conc
        assert sel.sum() > 50 and (got["mate_mapq"][:, sel] <= 1).all()
        assert (got["second_pair_score"][sel] == got["pair_score"][sel]).all()
        # one mate in the four-copy unit, its partner unique: the pair (mostly rescued: the repeat mate's own best lies in another copy)
        # is placed uniquely, the repeat mate alone is not
        sel = (kind == 2) & (got["pair_flags"] != 0)
        rm = np.where(repeat_mate == 1, 1, 0)
        single = se_mapq[rm, np.arange(n)]
        assert sel.sum() > 50 and (single[sel] <= 1).mean() > 0.9 and (got["mate_mapq"][0, sel] >= 30).mean() > 0.9
        # the 200-copy unit: long candidate lists
        assert (got["second_pair_score"][kind == 5] != INT_MIN).sum() > 30


def test_paired_mapq_quality_scheme(setup):
    """nvBowtie's quality-dependent scoring (d_read_quals) through the paired stage"""
    O, g, gw, idx, fmi = setup
    reads, _ = make_pairs(g, seed=33)
    rng = np.random.default_rng(9)
    quals = [rng.integers(0, 50, len(r)).astype(np.uint8) for r in reads]
    rs = packed(reads)
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    params = se_params(scheme=sch, read_quals=torch.from_numpy(np.concatenate(quals)).cuda())
    check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, nb.PairParams(min_frag=0, max_frag=400, min_mate_score=60), MapqParams.local(L),
                    quals=quals)


def test_paired_mapq_short_rescue_capacity(setup):
    """rescue_capacity below the jobs wanted: only the jobs run are candidates"""
    O, g, gw, idx, fmi = setup
    reads, _ = make_pairs(g, seed=55)
    rs = packed(reads)
    params = se_params()
    wanted = int(run(fmi, gw, rs, params, nb.PairParams(min_frag=0, max_frag=400, min_mate_score=60)).n_rescue[1])
    assert wanted > 20
    pair = nb.PairParams(min_frag=0, max_frag=400, min_mate_score=60, rescue_capacity=wanted // 2)
    got, _ = check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, pair, MapqParams.local(L))
    assert tuple(got["n_rescue"]) == (wanted // 2, wanted)


def test_paired_mapq_same_on_every_path(setup):
    """per-read and per-hit paths, the exact shortcut on and off, job de-duplication on and off, the one- and two-pass seed match, and
    the located k-mer table with and without the per-row context array: every output, old and new, identical"""
    O, g, gw, idx, fmi_s = setup
    L_ = nb.lib()
    reads, _ = make_pairs(g, n_pairs=3000, ragged=True, seed=77)
    rs = packed(reads)
    params = se_params()
    pair = nb.PairParams(min_frag=0, max_frag=400, min_mate_score=60)
    mq = MapqParams.local(L)
    fmi = nb.FMIndexDevice.from_text(gw, N_GENOME, sa_interval=1)[0]
    fmi.build_ktab(8, located=True, text=gw)
    assert fmi.rows is not None
    ref = outputs(run(fmi, gw, rs, params, pair, mq))
    assert (ref["second_pair_score"] != INT_MIN).sum() > 300

    def same(ws, what):
        got = outputs(ws)
        for k in got:
            assert np.array_equal(got[k][:2] if k == "n_hits" else got[k], ref[k][:2] if k == "n_hits" else ref[k]), (what, k)

    same(run(fmi_s, gw, rs, params, pair, mq), "sampled suffix array")
    rows = fmi.rows
    fmi.rows = None
    try:
        same(run(fmi, gw, rs, params, pair, mq), "without the per-row context array")
    finally:
        fmi.rows = rows
    for hook, off, on in ((L_.nvb_debug_pipeline_path, 1, 0), (L_.nvb_debug_perfect_shortcut, 0, 1), (L_.nvb_debug_seed_split, 0, 1)):
        hook(C.c_int(off))
        try:
            same(run(fmi, gw, rs, params, pair, mq), hook.__name__)
        finally:
            hook(C.c_int(on))
    params.dedup_jobs = False
    same(run(fmi, gw, rs, params, pair, mq), "dedup off")
    params.dedup_jobs = True
    # a workspace made without MAPQ outputs refuses them
    ws = run(fmi, gw, rs, params, pair)
    with pytest.raises(ValueError):
        nb.seed_extend_paired(fmi, gw, rs, params, pair, workspace=ws, mapq=mq)
