"""CPU: the paired MAPQ and second-best pair rule of nvb_seed_extend_paired_mapq, compiled for the host by tests/host/pair_mapq_harness.cu:
the MAPQ (and its numpy restatement) against nvBowtie's own BowtieMapq2 on paired alignments (tests/golden/mapq_paired.npz, written from
the reference by tests/golden/make_mapq_paired_golden.py), the pair rule against a brute-force Python restatement (tests/pair_mapq_oracle.py)
on random and hand-built candidate sets, and the entry point's argument validation."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle.ref_mapq import RefMapq
from oracle.ref_mapq_paired import RefMapqPaired
from tests.golden.make_mapq_paired_golden import pair_grid, configs
from tests.mapq_oracle import bowtie_mapq2
from tests.pair_mapq_oracle import second_pair

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "mapq_paired.npz")
SO = os.path.join(HERE, "host", "libpair_mapq_harness.so")
SRC = os.path.join(HERE, "host", "pair_mapq_harness.cu")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def G():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    return C.CDLL(SO)


def grid_points(G):
    """every fixture point as flat arrays (s1, s2, kind, t1, t2, len1, len2, match_bonus, min1, min2) and the fixture's MAPQ"""
    cols = [[] for _ in range(10)]
    for l1, l2, bonus, m1, m2, _ in G["cfg"]:
        pts = pair_grid(l1, l2, bonus, m1, m2)
        n = len(pts[0])
        for c, v in zip(cols, pts + (np.full(n, l1, np.uint32), np.full(n, l2, np.uint32), np.full(n, bonus, np.int32),
                                     np.full(n, m1, np.int32), np.full(n, m2, np.int32))):
            c.append(v)
    return [np.concatenate(c) for c in cols], G["mapq"]


def test_fixture_covers_the_grid(G):
    assert G["offsets"][-1] == len(G["mapq"]) > 2_000_000
    for c, (l1, l2, bonus, m1, m2, _) in enumerate(G["cfg"]):
        assert G["offsets"][c + 1] - G["offsets"][c] == len(pair_grid(l1, l2, bonus, m1, m2)[0])
    from nvbio_b200.pipeline import simple_func
    assert np.array_equal(configs(simple_func), G["cfg"])             # the host --score-min helper gives the fixture's min scores
    assert {int(v) for v in G["cfg"][:, 2]} == {0, 2, 3} and len({int(v) for v in G["cfg"][:, 5]}) == 8 and G["cfg"][:, :2].max() == 1000
    (s1, s2, kind, *_), want = grid_points(G)
    assert set(np.unique(kind)) == {0, 1, 2} and len(np.unique(want)) >= 40


def test_unpaired_second_counts_as_none(G):
    """in the reference an unpaired second alignment behind a paired best is no second at all"""
    (s1, s2, kind, t1, t2, l1, l2, bonus, m1, m2), want = grid_points(G)
    none = np.flatnonzero(kind == 0)
    owner = none[np.searchsorted(none, np.arange(len(kind)), side="right") - 1]      # each point's "no second" point (same best)
    assert np.array_equal(want[kind == 2], want[owner[kind == 2]])


def test_host_build_equals_reference(G, H):
    cols, want = grid_points(G)
    got = np.zeros(len(want), np.uint8)
    H.hh_bowtie_mapq2_paired(*[_p(np.ascontiguousarray(c)) for c in cols], C.c_uint32(len(want)), _p(got))
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [tuple(int(c[i]) for c in cols) + (int(got[i]), int(want[i])) for i in bad[:5]]


def test_python_restatement_equals_reference(G):
    (s1, s2, kind, t1, t2, l1, l2, bonus, m1, m2), want = grid_points(G)
    s1, s2, t1, t2, m1, m2 = (v.astype(np.int64) for v in (s1, s2, t1, t2, m1, m2))
    got = bowtie_mapq2(s1 + s2, kind == 1, t1 + t2, l1.astype(np.int64) + l2, bonus, m1 + m2)
    assert np.array_equal(got, want)


@pytest.mark.skipif(not (RefMapq.available() and RefMapqPaired.available()),
                    reason="oracle/_ref/libnvbio_ref_mapq{,_paired}.so (the reference's own code) are not built here")
def test_fixture_equals_live_reference(G):
    (s1, s2, kind, t1, t2, l1, l2, bonus, m1, m2), want = grid_points(G)
    assert np.array_equal(RefMapqPaired().mapq_paired(s1, s2, kind, t1, t2, l1, l2, bonus, m1, m2), want)
    assert np.array_equal(configs(RefMapq().simple_func), G["cfg"])


# ---- the pair rule ----------------------------------------------------------------------------------------------------------------

def merged(cands):
    """what pair_cand_merge_kernel leaves of a mate's candidates: sorted by (strand, end), one per (strand, end) -- the highest (score, -tie)"""
    best = {}
    for s, t, e, i in cands:
        k = (t, e)
        if k not in best or (s, -i) > (best[k][0], -best[k][1]):
            best[k] = (s, i)
    keys = sorted(best)
    return [(best[k][0], k[0], k[1], best[k][1]) for k in keys], sum(1 for k in keys if k[0] == 0)


def run_host(H, cases, min_frag, max_frag):
    """cases: (c1, c2, len1, len2, star, rescues) with the raw candidates (score, strand, end, tie) that reach the min score"""
    n = len(cases)
    seg, nfw, cnt, ln, end, score, tie, se, st = ([] for _ in range(9))
    mates = [[], []]
    for c1, c2, l1, l2, star, _ in cases:
        mates[0].append((c1, l1, star[0])); mates[1].append((c2, l2, star[1]))
    for m in range(2):
        for c, length, s in mates[m]:
            mc, fw = merged(c)
            seg.append(len(end)); nfw.append(fw); cnt.append(len(mc)); ln.append(length); se.append(s[0]); st.append(s[1])
            for sc, _, e, i in mc:
                end.append(e); score.append(sc); tie.append(i)
    nres = [len(c[5]) for c in cases]
    rz = [[0] * (2 * n) for _ in range(6)]
    for p, c in enumerate(cases):
        for k, r in enumerate(c[5]):
            for f in range(6):
                rz[f][2 * p + k] = r[f]
    u32 = lambda v: np.ascontiguousarray(v, np.uint32)      # noqa: E731
    i32 = lambda v: np.ascontiguousarray(v, np.int32)       # noqa: E731
    has = np.zeros(n, np.uint8); osc = np.zeros(n, np.int32); oend = np.zeros(2 * n, np.uint32); ost = np.zeros(2 * n, np.uint32)
    args = [u32(seg), u32(nfw), u32(cnt), u32(ln), u32(end + [0]), i32(score + [0]), u32(tie + [0]), u32(se), u32(st)]
    rargs = [u32(nres), u32(rz[0]), i32(rz[1]), u32(rz[2]), u32(rz[3]), u32(rz[4]), u32(rz[5])]
    H.hh_pair_second(C.c_uint32(n), *[_p(a) for a in args], C.c_uint32(min_frag), C.c_uint32(max_frag), *[_p(a) for a in rargs],
                     _p(has), _p(osc), _p(oend), _p(ost))
    out = []
    for p in range(n):
        out.append(None if not has[p] else (int(osc[p]), ((int(oend[p]), int(ost[p])), (int(oend[n + p]), int(ost[n + p])))))
    return out


def check(H, cases, min_frag, max_frag, min_score=None):
    """min_score: drop the candidates below it first, as pair_cand_scatter_kernel does"""
    if min_score is not None:
        cases = [([c for c in c1 if c[0] >= min_score], [c for c in c2 if c[0] >= min_score]) + tuple(rest) for c1, c2, *rest in cases]
    got = run_host(H, cases, min_frag, max_frag)
    for p, (c1, c2, l1, l2, star, resc) in enumerate(cases):
        want = second_pair(c1, c2, l1, l2, star, min_frag, max_frag, resc)
        assert got[p] == want, (p, c1, c2, l1, l2, star, resc, got[p], want)
    return got


def random_case(rng, span, lens):
    l1, l2 = (int(rng.choice(lens)) for _ in range(2))
    ties = iter(rng.permutation(100_000))

    def cands(length):
        c = []
        for _ in range(int(rng.integers(0, 9))):
            e = int(rng.integers(0, span))
            c.append((int(rng.integers(4, 9)) * 4, int(rng.integers(0, 2)), e, int(next(ties))))      # 16: below the min score
            if rng.random() < 0.2:                                          # the same (strand, end) again: merged
                c.append((c[-1][0] - 4 * int(rng.integers(0, 2)), c[-1][1], e, int(next(ties))))
        return c
    c1, c2 = cands(l1), cands(l2)
    star = []
    for c, length in ((c1, l1), (c2, l2)):
        if c and rng.random() < 0.7:
            s, t, e, _ = c[int(rng.integers(0, len(c)))]
            star.append((e + int(rng.choice([0, 0, length // 2, length // 2 + 1, -(length // 2), -(length // 2) - 1])), t))
        else:
            star.append((int(rng.integers(0, span)), int(rng.integers(0, 2))))
    star[0] = (max(star[0][0], 0), star[0][1]); star[1] = (max(star[1][0], 0), star[1][1])
    resc = []
    for a in range(2):
        if rng.random() < 0.3:
            oe = int(rng.integers(0, span))
            ae, at = star[a] if rng.random() < 0.5 else (int(rng.integers(0, span)), int(rng.integers(0, 2)))
            resc.append((a, int(rng.integers(10, 17)) * 4, ae, at, int(next(ties)), oe))
    return (c1, c2, l1, l2, tuple(star), resc)


@pytest.mark.parametrize("min_frag,max_frag", [(0, 120), (40, 90), (0, 0xFFFFFFFF - 5)])
def test_pair_rule_random(H, min_frag, max_frag):
    rng = np.random.default_rng(min_frag * 7 + max_frag % 1000)
    cases = [random_case(rng, 260, (10, 11, 30, 31, 60)) for _ in range(4000)]
    got = check(H, cases, min_frag, max_frag, min_score=20)
    assert sum(g is not None for g in got) > 1000 and sum(g is None for g in got) > 100


def test_pair_rule_edges(H):
    """hand-built edges of the rule: fragments exactly at min_frag / max_frag, forward end equal to reverse end, begins clamped at 0,
    neighbours at len/2 and len/2 + 1 of P*, exact ties, rescue-only pairs, both rescues tying, a combination scoring above P*"""
    L, MIN, MAX = 20, 30, 60
    star = ((100, 0), (140, 1))                                               # P*: mate 1 forward [80, 100), mate 2 reverse [120, 140)
    cases, want_scores = [], []

    def case(c1, c2, resc=(), st=star, want=None):
        cases.append((c1, c2, L, L, st, list(resc))); want_scores.append(want)
    # fragment exactly max_frag (re - fb = 60) and max_frag + 1; exactly min_frag and min_frag - 1 (fb = 300 - 20 = 280)
    case([(40, 0, 300, 1)], [(40, 1, 340, 2)], want=80)
    case([(40, 0, 300, 1)], [(40, 1, 341, 2)], want=None)
    case([(40, 0, 300, 1)], [(40, 1, 310, 2)], want=80)
    case([(40, 0, 300, 1)], [(40, 1, 309, 2)], want=None)
    # forward end == reverse end (fragment = L): needs min_frag <= 20
    cases_eq = [([(40, 0, 300, 1)], [(40, 1, 300, 2)], L, L, star, [])]
    # begins clamped at 0: forward mate ending at 5 begins at 0; reverse ending at 25 begins at 5 >= 0
    cases_clamp = [([(40, 0, 5, 1)], [(40, 1, 25, 2)], L, L, star, []), ([(40, 1, 25, 1)], [(40, 0, 5, 2)], L, L, star, [])]
    # not distinct at len/2 on both mates (not a second pair); one mate at len/2 + 1 (distinct)
    case([(40, 0, 100 + L // 2, 1)], [(40, 1, 140 - L // 2, 2)], want=None)
    case([(40, 0, 100 + L // 2 + 1, 1)], [(40, 1, 140, 2)], want=80)
    case([(40, 0, 100, 1)], [(40, 1, 140 - L // 2 - 1, 2)], want=80)
    # exact ties: the smaller mate-1 tie index, then the smaller mate-2 tie index
    case([(40, 0, 300, 7), (40, 0, 500, 3)], [(40, 1, 330, 1), (40, 1, 530, 9)], want=80)
    case([(40, 0, 300, 3), (40, 0, 301, 4)], [(40, 1, 330, 8), (40, 1, 331, 2)], want=80)
    # rescue-only (no candidates), both rescues tying (mate 1 as anchor wins), a rescue tying a combination with the same mate-1 tie
    # index (the combination wins: the rescued mate's tie index is 0xFFFFFFFF)
    case([], [], resc=[(0, 90, 300, 0, 5, 340)], want=90)
    case([], [], resc=[(0, 90, 300, 0, 5, 340), (1, 90, 600, 1, 2, 560)], want=90)
    case([(45, 0, 700, 5)], [(45, 1, 740, 9)], resc=[(0, 90, 300, 0, 5, 340)], want=90)
    # a distinct combination scoring above P* is still the second pair
    case([(70, 0, 300, 1)], [(70, 1, 340, 2)], want=140)
    got = check(H, cases, MIN, MAX)
    for g, w in zip(got, want_scores):
        assert (g is None and w is None) or (g is not None and g[0] == w), (g, w)
    assert got[-4][1] == ((300, 0), (340, 1)) and got[-3][1] == ((300, 0), (340, 1))      # anchors' ties
    assert got[-2][1] == ((700, 0), (740, 1)) and got[7][1] == ((500, 0), (530, 1)) and got[8][1] == ((300, 0), (331, 1))
    assert check(H, cases_eq, 0, MAX)[0][0] == 80 and check(H, cases_eq, L + 1, MAX)[0] is None
    assert [g[0] for g in check(H, cases_clamp, 0, MAX)] == [80, 80]


def test_argument_validation_without_gpu():
    """nvb_seed_extend_paired_mapq rejects missing MAPQ inputs / outputs, a min-score table shorter than the reads and what
    nvb_seed_extend_paired rejects with NVB_E_INVALID (-1) before any CUDA call, also when the reads would be NVB_E_UNSUPPORTED (-4)"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, SeedExtendParamsStruct, FmIndexStruct, MapqParamsStruct,
                                 PairParamsStruct, PairOutStruct, PairMapqOutStruct)
    L = _lib.lib()
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    tb = C.c_size_t(0)

    def good():
        pp = PairParamsStruct(); pp.min_frag, pp.max_frag, pp.min_mate_score, pp.rescue_capacity = 0, 500, 60, 8
        po = PairOutStruct(); po.d_pair_score = po.d_pair_flags = po.d_mate_score = po.d_mate_pos = po.d_mate_strand = 16
        mp = MapqParamsStruct(); mp.d_min_score, mp.max_read_len, mp.match_bonus = 16, 150, 2
        mo = PairMapqOutStruct(); mo.d_second_pair_score, mo.d_mate_mapq = 16, 16
        return pp, po, mp, mo

    def call(pp, po, mp, mo, n_pairs=4, reads=ss, params=sp, temp_bytes=tb):
        r = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return L.nvb_seed_extend_paired_mapq(C.byref(fm), C.c_void_p(16), r(reads), C.c_uint32(n_pairs), r(params), C.c_uint32(100),
                                             r(pp), r(po), r(mp), r(mo), None, None, r(temp_bytes), None)

    pp, po, mp, mo = good()
    assert call(None, po, mp, mo) == -1 and call(pp, None, mp, mo) == -1 and call(pp, po, None, mo) == -1 and call(pp, po, mp, None) == -1
    pp, po, mp, mo = good(); mp.d_min_score = None; assert call(pp, po, mp, mo) == -1
    for field in ("d_second_pair_score", "d_mate_mapq"):
        pp, po, mp, mo = good(); setattr(mo, field, None); assert call(pp, po, mp, mo) == -1
    pp, po, mp, mo = good(); mp.max_read_len = 149; assert call(pp, po, mp, mo) == -1
    for field in ("d_pair_score", "d_mate_pos"):
        pp, po, mp, mo = good(); setattr(po, field, None); assert call(pp, po, mp, mo) == -1
    pp, po, mp, mo = good(); pp.min_frag = 600; assert call(pp, po, mp, mo) == -1
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, n_pairs=0x40000000) == -1
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, reads=None) == -1 and call(pp, po, mp, mo, temp_bytes=None) == -1
    # 8-bit reads are NVB_E_UNSUPPORTED (-4), but every failed pair or MAPQ check wins over it
    s8 = StringSetStruct(); s8.d_words = 16; s8.bits = 8; s8.big_endian = 1; s8.stride = 152; s8.length = 150
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, reads=s8) == -4
    pp, po, mp, mo = good(); mp.max_read_len = 149; assert call(pp, po, mp, mo, reads=s8) == -1
    pp, po, mp, mo = good(); mo.d_mate_mapq = None; assert call(pp, po, mp, mo, reads=s8) == -1
    pp, po, mp, mo = good(); assert call(pp, po, None, mo, reads=s8) == -1 and call(pp, po, mp, None, reads=s8) == -1
    pp, po, mp, mo = good(); po.d_mate_strand = None; assert call(pp, po, mp, mo, reads=s8) == -1
    pp, po, mp, mo = good(); pp.max_frag = 0; assert call(pp, po, mp, mo, reads=s8) == -1
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, reads=s8, temp_bytes=None) == -1
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, reads=s8, n_pairs=0x40000000) == -1
    one = SeedExtendParamsStruct(); one.seed_len, one.seed_interval, one.band_len, one.type, one.both_strands, one.max_seed_hits = 20, 10, 31, 1, 0, 100
    one.scheme = sch
    pp, po, mp, mo = good(); assert call(pp, po, mp, mo, reads=s8, params=one) == -1 and call(pp, po, mp, mo, params=None) == -1
    # the paired traceback's 512 bp limit does not apply here: reads of 513 bp reach the seed checks
    s513 = StringSetStruct(); s513.d_words = 16; s513.bits = 2; s513.big_endian = 1; s513.stride = 528; s513.length = 513
    no_seed = SeedExtendParamsStruct(); no_seed.seed_len, no_seed.seed_interval, no_seed.band_len, no_seed.type = 0, 10, 31, 1
    no_seed.both_strands, no_seed.max_seed_hits, no_seed.dedup_jobs, no_seed.scheme = 1, 100, 1, sch
    pp, po, mp, mo = good(); mp.max_read_len = 513; assert call(pp, po, mp, mo, reads=s513, params=no_seed) == -1
