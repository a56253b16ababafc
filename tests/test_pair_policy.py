"""CPU: the paired-end policies of seed + extend (nvb_pair_params.policy / flags), compiled for the host by
tests/host/pair_policy_harness.cu: the framing against nvBowtie's own frame_opposite_mate (oracle/_ref where it is built, else
tests/golden/pe_policy.npz, written from the reference by tests/golden/make_pe_policy_golden.py), the concordance test and the rescue
window against their Python restatements (tests/pair_policy_oracle.py) and the FR rules they replace, the general pair_combinations
against a brute force over every combination, the policy oracles at their defaults against the FR oracles they generalise, and the
entry points' argument validation."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle.ref_pe_policy import RefPePolicy
from tests.golden.make_pe_policy_golden import inputs
from tests.pair_policy_oracle import frame, concordant, rescue_window, second_pair
from tests.test_pair_mapq import merged

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "pe_policy.npz")
SO = os.path.join(HERE, "host", "libpair_policy_harness.so")
SRC = os.path.join(HERE, "host", "pair_policy_harness.cu")
POLICIES = ("fr", "rf", "ff", "rr")                 # NVB_PE_* numbering
REF_NUM = {"ff": 0, "fr": 1, "rf": 2, "rr": 3}      # io::PE_POLICY_* numbering
NO_OVERLAP = 1
FLAG_SETS = (0, 1, 2, 4, 7)                        # the framing rules read NO_OVERLAP only; the other bits must not change them


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def u32(v):
    return np.ascontiguousarray(v, np.uint32)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "pipeline_core.cuh", "common.cuh")]
    deps.append(os.path.join(HERE, "..", "include", "nvbio_b200.h"))
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    return C.CDLL(SO)


def host_frame(H, policy, a, t):
    n = len(policy)
    left, strand = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    H.hp_frame(_p(u32(policy)), _p(u32(a)), _p(u32(t)), C.c_uint32(n), _p(left), _p(strand))
    return left, strand


def host_concordant(H, policy, flags, min_frag, max_frag, m1, m2):
    """m1 / m2: (t, b, e) arrays"""
    n = len(m1[0])
    out = np.zeros(n, np.uint8)
    H.hp_concordant(C.c_uint32(POLICIES.index(policy)), C.c_uint32(flags), C.c_uint32(min_frag), C.c_uint32(max_frag),
                    *[_p(u32(v)) for v in tuple(m1) + tuple(m2)], C.c_uint32(n), _p(out))
    return out.astype(bool)


# ---- framing --------------------------------------------------------------------------------------------------------------------

def reference_frames():
    """(policy, anchor, anchor_fw, left, fw) of nvBowtie's frame_opposite_mate on all 16 inputs: live where oracle/_ref is built"""
    if RefPePolicy.available():
        policy, anchor, anchor_fw = inputs()
        left, fw = RefPePolicy().frame(policy, anchor, anchor_fw)
        return policy, anchor, anchor_fw, left, fw
    G = np.load(GOLDEN)
    return G["policy"], G["anchor"], G["anchor_fw"], G["left"], G["fw"]


def test_frame_equals_reference(H):
    policy, anchor, anchor_fw, left, fw = reference_frames()
    assert len(policy) == 16 and len({(int(p), int(a), int(f)) for p, a, f in zip(policy, anchor, anchor_fw)}) == 16
    ours = np.array([POLICIES.index({v: k for k, v in REF_NUM.items()}[int(p)]) for p in policy], np.uint32)
    t = 1 - anchor_fw.astype(np.uint32)                             # anchor_fw = (t == 0)
    hl, hs = host_frame(H, ours, anchor, t)
    assert np.array_equal(hl, left) and np.array_equal(hs, 1 - fw)
    for i in range(16):                                             # the Python restatement the oracles use
        assert frame(POLICIES[ours[i]], int(anchor[i]), int(t[i])) == (bool(left[i]), 1 - int(fw[i]))


@pytest.mark.skipif(not RefPePolicy.available(), reason="oracle/_ref/libnvbio_ref_pe_policy.so (the reference's own code) is not built here")
def test_fixture_equals_live_reference():
    policy, anchor, anchor_fw = inputs()
    left, fw = RefPePolicy().frame(policy, anchor, anchor_fw)
    G = np.load(GOLDEN)
    assert np.array_equal(G["policy"], policy) and np.array_equal(G["left"], left) and np.array_equal(G["fw"], fw)


# ---- concordance ----------------------------------------------------------------------------------------------------------------

def random_mates(rng, n, span=400, lens=(1, 20, 50, 51, 100)):
    """(t, b, e) of n random mates with begins clamped at 0 and many equal begins / ends"""
    ln = rng.choice(lens, n)
    e = rng.integers(0, span, n)
    e = np.where(rng.random(n) < 0.1, rng.integers(0, 3, n), e)           # ends near 0: begins clamped
    return rng.integers(0, 2, n), np.maximum(e - ln, 0), e


def fr_before(m1, m2, min_frag, max_frag):
    """nvb_seed_extend_paired's original FR test (fr_concordant over the forward / reverse mate)"""
    t1, b1, e1 = (v.astype(np.int64) for v in m1)
    t2, b2, e2 = (v.astype(np.int64) for v in m2)
    fw1 = t1 == 0
    fb, fe, rb, re_ = np.where(fw1, b1, b2), np.where(fw1, e1, e2), np.where(fw1, b2, b1), np.where(fw1, e2, e1)
    return (t1 != t2) & (fb <= rb) & (fe <= re_) & (re_ > fb) & (re_ - fb >= min_frag) & (re_ - fb <= max_frag)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("flags", FLAG_SETS)
def test_concordance_is_symmetric_and_equals_restatement(H, policy, flags):
    rng = np.random.default_rng(POLICIES.index(policy) * 31 + flags)
    n, min_frag, max_frag = 60_000, 30, 150
    m1, m2 = random_mates(rng, n), random_mates(rng, n)
    got = host_concordant(H, policy, flags, min_frag, max_frag, m1, m2)
    assert got.sum() > 500 and (~got).sum() > 500
    # framing from mate 2: the same mates with mate 2 as "mate 1" of the reversed policy view
    for i in np.flatnonzero(got)[:2000].tolist() + np.flatnonzero(~got)[:2000].tolist():
        a, b = tuple(int(v[i]) for v in m1), tuple(int(v[i]) for v in m2)
        want = concordant(policy, not (flags & NO_OVERLAP), a, b, min_frag, max_frag)
        assert got[i] == want, (policy, flags, a, b)
        left2, o2 = frame(policy, 1, b[0])
        sym = a[0] == o2
        if sym:
            (_, lb, le), (_, rb, re_) = (a, b) if left2 else (b, a)
            sym = lb <= rb and le <= re_ and re_ > lb and min_frag <= re_ - lb <= max_frag and (not (flags & NO_OVERLAP) or le <= rb)
        assert sym == want, (policy, flags, a, b)


def test_concordance_fr_equals_the_rule_it_replaces(H):
    rng = np.random.default_rng(7)
    n = 1_200_000
    for min_frag, max_frag in ((0, 500), (30, 150), (0, 0xFFFFFFFF - 3)):
        m1, m2 = random_mates(rng, n, span=700), random_mates(rng, n, span=700)
        got = host_concordant(H, "fr", 0, min_frag, max_frag, m1, m2)
        assert np.array_equal(got, fr_before(m1, m2, min_frag, max_frag))
        assert got.sum() > 10_000


def test_concordance_edges(H):
    """equal begins and ends, a begin clamped at 0, fragments of exactly min_frag / max_frag and one past, L.e == R.b"""
    cases = []                                                      # (policy, flags, mate 1 (t, b, e), mate 2, min, max, want)
    for policy in POLICIES:
        for a_t in (0, 1):
            left, o = frame(policy, 0, a_t)

            def mk(lb, le, rb, re_):                                 # mate 1 / mate 2 laid out as framed from mate 1
                return ((a_t, rb, re_), (o, lb, le)) if left else ((a_t, lb, le), (o, rb, re_))
            cases += [(policy, 0) + mk(100, 120, 100, 120) + (0, 60, True),          # equal begins and ends: fragment = L
                      (policy, 0) + mk(100, 120, 100, 120) + (21, 60, False),
                      (policy, 1) + mk(100, 120, 100, 120) + (0, 60, False),          # ... overlap
                      (policy, 0) + mk(0, 5, 5, 25) + (0, 60, True),                  # begin clamped at 0
                      (policy, 0) + mk(100, 120, 140, 160) + (60, 60, True),          # exactly min_frag = max_frag
                      (policy, 0) + mk(100, 120, 141, 161) + (0, 60, False),          # max_frag + 1
                      (policy, 0) + mk(100, 120, 139, 159) + (60, 90, False),         # min_frag - 1
                      (policy, 1) + mk(100, 120, 120, 140) + (0, 60, True),           # L.e == R.b
                      (policy, 1) + mk(100, 121, 120, 140) + (0, 60, False),          # L.e == R.b + 1
                      (policy, 0) + mk(100, 121, 120, 140) + (0, 60, True),
                      (policy, 0) + mk(101, 120, 100, 140) + (0, 60, False),          # L begins after R
                      (policy, 0) + mk(100, 141, 100, 140) + (0, 60, False)]          # L ends after R
            bad_strand = mk(100, 120, 140, 160)
            cases.append((policy, 0, bad_strand[0], (1 - o,) + bad_strand[1][1:], 0, 60, False))
    for policy, flags, m1, m2, mn, mx, want in cases:
        got = host_concordant(H, policy, flags, mn, mx, [np.array([v]) for v in m1], [np.array([v]) for v in m2])[0]
        assert got == want == concordant(policy, not (flags & NO_OVERLAP), m1, m2, mn, mx), (policy, flags, m1, m2, mn, mx)
        assert concordant(policy, not (flags & NO_OVERLAP), m1, m2, mn, mx) == want


# ---- rescue window --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("flags", FLAG_SETS)
def test_rescue_window_matches_table(H, policy, flags):
    rng = np.random.default_rng(POLICIES.index(policy) * 7 + flags + 100)
    n, glen = 50_000, 5_000
    for max_frag in (1, 300, 6_000, 0xFFFFFFFF):
        a, t = rng.integers(0, 2, n), rng.integers(0, 2, n)
        e = rng.integers(0, glen + 1, n)
        e = np.where(rng.random(n) < 0.1, rng.integers(glen - 3, glen + 1, n), e)
        b = np.maximum(e - rng.choice((1, 20, 100), n), 0)
        wb, wl, ws = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        H.hp_rescue_window(C.c_uint32(POLICIES.index(policy)), C.c_uint32(flags), C.c_uint32(max_frag), C.c_uint32(glen),
                           *[_p(u32(v)) for v in (a, t, b, e)], C.c_uint32(n), _p(wb), _p(wl), _p(ws))
        for i in range(0, n, 7):
            w0, w1, o = rescue_window(policy, not (flags & NO_OVERLAP), int(a[i]), int(t[i]), int(b[i]), int(e[i]), max_frag, glen)
            assert (int(wb[i]), int(wl[i]), int(ws[i])) == (w0, w1 - w0, o), (i, int(a[i]), int(t[i]), int(b[i]), int(e[i]), max_frag)
        if policy == "fr" and flags in (0, 2, 4):                    # the rule it replaces (pair_classify_kernel before policies)
            fw = t == 0
            to = np.where(fw, b, np.where(e > max_frag, e - max_frag, 0)).astype(np.int64)
            te = np.where(fw, np.minimum(b.astype(np.int64) + max_frag, glen), e)
            assert np.array_equal(wb, to) and np.array_equal(wl, te - to) and np.array_equal(ws, 1 - t)


# ---- second-best pair over the concordant combinations ----------------------------------------------------------------------------

def run_combinations(H, cases, policy, flags, min_frag, max_frag):
    n = len(cases)
    seg, nfw, cnt, ln, end, score, tie, se, st = ([] for _ in range(9))
    mates = [[], []]
    for c1, c2, l1, l2, star in cases:
        mates[0].append((c1, l1, star[0])); mates[1].append((c2, l2, star[1]))
    for m in range(2):
        for c, length, s in mates[m]:
            mc, fw = merged(c)
            seg.append(len(end)); nfw.append(fw); cnt.append(len(mc)); ln.append(length); se.append(s[0]); st.append(s[1])
            for sc, _, e, i in mc:
                end.append(e); score.append(sc); tie.append(i)
    has = np.zeros(n, np.uint8); osc = np.zeros(n, np.int32); oend = np.zeros(2 * n, np.uint32); ost = np.zeros(2 * n, np.uint32)
    args = [u32(seg), u32(nfw), u32(cnt), u32(ln), u32(end + [0]), np.ascontiguousarray(score + [0], np.int32), u32(tie + [0]), u32(se), u32(st)]
    H.hp_pair_combinations(C.c_uint32(n), C.c_uint32(POLICIES.index(policy)), C.c_uint32(flags), *[_p(a) for a in args],
                           C.c_uint32(min_frag), C.c_uint32(max_frag), _p(has), _p(osc), _p(oend), _p(ost))
    return [None if not has[p] else (int(osc[p]), ((int(oend[p]), int(ost[p])), (int(oend[n + p]), int(ost[n + p])))) for p in range(n)]


def random_cands(rng, span, length, ties):
    c = []
    for _ in range(int(rng.integers(0, 10))):
        e = int(rng.integers(0, span)) if rng.random() > 0.1 else int(rng.integers(0, 4))    # some begins clamped at 0
        c.append((int(rng.integers(5, 9)) * 4, int(rng.integers(0, 2)), e, int(next(ties))))
        if rng.random() < 0.2:                                      # the same (strand, end) again: merged
            c.append((c[-1][0] - 4 * int(rng.integers(0, 2)), c[-1][1], e, int(next(ties))))
        if rng.random() < 0.15:                                     # an equal score elsewhere: ties
            c.append((c[-1][0], int(rng.integers(0, 2)), int(rng.integers(0, span)), int(next(ties))))
    return c


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("flags", (0, NO_OVERLAP))
def test_pair_combinations_equal_brute_force(H, policy, flags):
    rng = np.random.default_rng(POLICIES.index(policy) * 3 + flags + 500)
    min_frag, max_frag, span = 10, 120, 260
    cases = []
    for _ in range(3000):
        ties = iter(rng.permutation(100_000))
        l1, l2 = (int(rng.choice((10, 11, 30, 31, 60))) for _ in range(2))
        c1, c2 = random_cands(rng, span, l1, ties), random_cands(rng, span, l2, ties)
        star = ((int(rng.integers(0, span)), int(rng.integers(0, 2))), (int(rng.integers(0, span)), int(rng.integers(0, 2))))
        cases.append((c1, c2, l1, l2, star))
    got = run_combinations(H, cases, policy, flags, min_frag, max_frag)
    for p, (c1, c2, l1, l2, star) in enumerate(cases):
        want = second_pair(c1, c2, l1, l2, star, min_frag, max_frag, (), policy, not (flags & NO_OVERLAP))
        assert got[p] == want, (policy, flags, c1, c2, l1, l2, star, got[p], want)
    assert sum(g is not None for g in got) > 500


# ---- argument validation ----------------------------------------------------------------------------------------------------------

def test_argument_validation_without_gpu():
    """a policy > 3 or an unknown flag bit fails in the four paired calls and in nvb_pipeline_create; NVB_PE_DISCORDANT fails without
    mapq / mapq_out in the paired calls and always in nvb_pipeline_create -- NVB_E_INVALID (-1) before any CUDA call"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, SeedExtendParamsStruct, FmIndexStruct, MapqParamsStruct,
                                 PairParamsStruct, PairOutStruct, PairMapqOutStruct, BestAlignmentOutStruct, ReseedParamsStruct)
    L = _lib.lib()
    # 8-bit reads are NVB_E_UNSUPPORTED (-4) after every pair check: a valid policy reaches it, an invalid one does not
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 8; ss.big_endian = 1; ss.stride = 152; ss.length = 150
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    po = PairOutStruct(); po.d_pair_score = po.d_pair_flags = po.d_mate_score = po.d_mate_pos = po.d_mate_strand = 16
    mp = MapqParamsStruct(); mp.d_min_score, mp.max_read_len, mp.match_bonus = 16, 150, 2
    mo = PairMapqOutStruct(); mo.d_second_pair_score, mo.d_mate_mapq = 16, 16
    ba = BestAlignmentOutStruct(); ba.d_ops, ba.max_ops, ba.d_n_ops, ba.d_begin = 16, 300, 16, 16
    rp = ReseedParamsStruct(); rp.max_reseed, rp.rep_seeds = 0, 300
    g = C.c_void_p(16)

    def pp(policy=0, flags=0):
        p = PairParamsStruct(); p.min_frag, p.max_frag, p.min_mate_score, p.rescue_capacity = 0, 500, 60, 8
        p.policy, p.flags = policy, flags
        return p

    def calls(p, with_mapq):
        m, o = (C.byref(mp), C.byref(mo)) if with_mapq else (None, None)
        tb = C.c_size_t(0)
        r = [L.nvb_seed_extend_paired(C.byref(fm), g, C.byref(ss), C.c_uint32(4), C.byref(sp), C.c_uint32(64), C.byref(p), C.byref(po),
                                      None, None, C.byref(tb), None),
             L.nvb_seed_extend_paired_traceback(C.byref(fm), g, C.byref(ss), C.c_uint32(4), C.byref(sp), C.c_uint32(64), C.byref(p),
                                                C.byref(po), C.byref(ba), m, o, None, None, C.byref(tb), None),
             L.nvb_seed_extend_paired_reseed(C.byref(fm), g, C.byref(ss), C.c_uint32(4), C.byref(sp), C.c_uint32(64), C.byref(p),
                                             C.byref(po), None, m, o, C.byref(rp), None, None, None, C.byref(tb), None)]
        if with_mapq:
            r.append(L.nvb_seed_extend_paired_mapq(C.byref(fm), g, C.byref(ss), C.c_uint32(4), C.byref(sp), C.c_uint32(64), C.byref(p),
                                                   C.byref(po), C.byref(mp), C.byref(mo), None, None, C.byref(tb), None))
        return r

    def create(p):
        out = C.c_void_p()
        return L.nvb_pipeline_create(C.byref(fm), g, C.byref(sp), C.byref(p), C.c_uint32(8), C.c_uint32(150), C.c_uint32(10), C.c_uint32(2),
                                     C.c_uint32(64), C.c_uint32(2), C.byref(out))

    for pol in range(4):
        for fl in (0, 1, 4, 5):
            assert all(r == -4 for r in calls(pp(pol, fl), True)), (pol, fl)
            assert all(r == -4 for r in calls(pp(pol, fl), False)), (pol, fl)
        for fl in (2, 7):                                          # the plain call has no MAPQ stage: discordant pairs always fail there
            r = calls(pp(pol, fl), True)
            assert r[0] == -1 and all(v == -4 for v in r[1:]), (pol, fl, r)
    for bad in (pp(4, 0), pp(0xFFFFFFFF, 0), pp(0, 8), pp(0, 0x80000000), pp(1, 0x10 | 1)):
        assert all(r == -1 for r in calls(bad, True)) and all(r == -1 for r in calls(bad, False))
        assert create(bad) == -1
    # discordant pairs need the MAPQ stage: the plain call always, _traceback / _reseed without mapq, the pipeline always
    for fl in (2, 3, 6, 7):
        assert all(r == -1 for r in calls(pp(1, fl), False))
        assert create(pp(0, fl)) == -1


# ---- the policy oracles at their defaults ---------------------------------------------------------------------------------------------

def test_policy_oracles_default_to_the_fr_oracles():
    """with a default PairParams (FR, overlap, no discordant pairs, mixed) the policy oracles give the FR oracles' outputs, field by field,
    single round and with reseeding rounds; with policy / options set they differ somewhere"""
    from oracle import orc
    from nvbio_b200 import aln
    from nvbio_b200.pipeline import SeedExtendParams, PairParams, simple_func
    from tests import pair_policy_oracle as ppo
    from tests.pipeline_oracle import seed_extend_paired_oracle
    from tests.pair_mapq_oracle import pair_mapq_oracle
    from tests.paired_reseed_oracle import seed_extend_paired_reseed_oracle, planted_pairs, RL, L, I
    O = orc.Oracle()
    g, reads, _, _ = planted_pairs(per_class=(4, 4, 8, 10, 8, 4, 10, 2))
    idx, n = O.build_index(g), len(reads) // 2
    ms = simple_func("G", 0.0, 10.0, np.arange(RL + 1))
    params = SeedExtendParams(seed_len=L, seed_interval=I, band_len=15, type=aln.LOCAL, both_strands=True, max_seed_hits=4,
                              scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    pair = PairParams(min_frag=0, max_frag=500, min_mate_score=60)

    def same(a, b):
        return all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a if k in b)
    assert same(ppo.seed_extend_paired_oracle(O, idx, g, reads, params, pair, n), seed_extend_paired_oracle(O, idx, g, reads, params, pair, n))
    want = pair_mapq_oracle(O, idx, g, reads, params, pair, n, ms, 2)
    assert same(ppo.pair_mapq_oracle(O, idx, g, reads, params, pair, n, ms, 2), want)
    assert same(ppo.seed_extend_paired_reseed_oracle(O, idx, g, reads, params, pair, n, 2, 8, 10**9, min_score=ms, match_bonus=2),
                seed_extend_paired_reseed_oracle(O, idx, g, reads, params, pair, n, 2, 8, 10**9, min_score=ms, match_bonus=2))
    other = PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy="rf", overlap=False, discordant=True, mixed=False)
    assert not same(ppo.pair_mapq_oracle(O, idx, g, reads, params, other, n, ms, 2), want)

