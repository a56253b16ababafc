"""-m gpu: banded Gotoh parity through the C ABI against the reference-generated golden fixtures and the
oracle; the packed DPX path and the generic int32 path are both exercised and compared with each other."""
import ctypes as C
import os
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.strings import PackedStringSet
from tests.gpu_util import require_gpu, host_u32
from tests.golden.make_golden import G1_P, G1_T, G2_P, G2_T, random_problems
from tests.test_host_core import fixed_problems

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def O():
    require_gpu()
    return orc.Oracle()


def force_path(p):
    nb.lib().nvb_debug_force_gotoh_path(C.c_int(p))


def run(band, typ, scheme, pr, pbits=4, tbits=8, pbe=True, tbe=False, quals=None, max_m=None):
    pat, p_off, p_len, txt, t_off, t_len = pr
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits, big_endian=pbe)
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=tbits, big_endian=tbe)
    if max_m is not None:
        P.length = max_m
    sch = scheme if not isinstance(scheme, tuple) else aln.SimpleGotohScheme(*scheme)
    q = torch.from_numpy(quals).cuda() if quals is not None else None
    s, k = aln.batch_banded_alignment_score(band, aln.make_gotoh_aligner(typ, sch), P, T, quals=q)
    torch.cuda.synchronize()
    k = host_u32(k)
    return s.cpu().numpy(), k[:, 0], k[:, 1]


def same(got, want):
    return all(np.array_equal(a, b) for a, b in zip(got, want[:3]))


def test_reference_asserted_problems(O):
    g = np.load(os.path.join(GOLD, "banded_gotoh.npz"))
    for name, P, T, scheme, band in (("g1", G1_P, G1_T, (2, -1, -1, -1), 7), ("g2", G2_P, G2_T, (0, -5, -8, -3), 31)):
        p, t = orc.dna(P), orc.dna(T)
        for typ in (0, 1, 2):
            for tbits in (2, 8):            # 2-bit text -> packed DPX path (when admissible), 8-bit -> generic
                s, x, y = run(band, typ, scheme, (p, [0], [len(p)], t, [0], [len(t)]), pbits=2, tbits=tbits, tbe=True)
                assert (int(s[0]), int(x[0]), int(y[0])) == tuple(int(v) for v in g[f"{name}_t{typ}"][:3]), (name, typ, tbits)


def test_golden_random(O):
    g = np.load(os.path.join(GOLD, "banded_gotoh.npz"))
    for cid, band, typ, m, mm, go, ge in g["cases"]:
        pr = [g[f"r{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len")]
        res = g[f"r{cid}_res"]
        s, x, y = run(int(band), int(typ), (int(m), int(mm), int(go), int(ge)), pr)
        assert np.array_equal(s.astype(np.int64), res[0]), (cid, band, typ)
        assert np.array_equal(x.astype(np.int64), res[1]) and np.array_equal(y.astype(np.int64), res[2]), (cid, band, typ)


@pytest.mark.parametrize("band", [7, 15, 31])
@pytest.mark.parametrize("typ", [0, 1, 2])
def test_packed_path_vs_oracle(O, band, typ):
    rng = np.random.default_rng(band * 7 + typ)
    for scheme in ((2, -2, -5, -3), (2, -1, -1, -1), (0, -5, -8, -3), (1, -3, -2, -4), (2, -6, -8, -3)):
        for ragged in (False, True):
            pr = fixed_problems(rng, 1037, band, 150, extra_text=int(rng.integers(0, 3)), ragged=ragged)
            want = O.banded_gotoh(band, typ, scheme, *pr)
            # little-endian patterns: refused by the DPX pair kernels' admission, scored by the generic kernel, the same results
            for pbits, tbe, pbe in ((2, True, True), (4, False, True), (2, True, False), (4, True, False)):
                force_path(0)
                assert same(run(band, typ, scheme, pr, pbits=pbits, tbits=2, pbe=pbe, tbe=tbe, max_m=150), want), (band, typ, scheme, ragged, pbe)
            # kernel variants: run-time pattern format instead of the compile-time 2- / 4-bit big-endian readers; one pattern row per
            # loop iteration instead of two in flight
            for fmt, rows2 in ((0, 1), (1, 0), (0, 0)):
                L = nb.lib()
                L.nvb_debug_pair_format(C.c_int(fmt)); L.nvb_debug_pair_rows2(C.c_int(rows2))
                try:
                    assert same(run(band, typ, scheme, pr, pbits=4, tbits=2, tbe=True, max_m=150), want), (band, typ, scheme, ragged, fmt, rows2)
                finally:
                    L.nvb_debug_pair_format(C.c_int(1)); L.nvb_debug_pair_rows2(C.c_int(1))
            force_path(1)
            try:
                assert same(run(band, typ, scheme, pr, pbits=2, tbits=2, tbe=True, max_m=150), want)
            finally:
                force_path(0)


def test_mixed_batch_fallback_list(O):
    """batches mixing admissible pairs with short windows / N's / empty patterns"""
    rng = np.random.default_rng(1)
    pr = random_problems(rng, 3001, 31, 150, alphabet_text=4)
    want = O.banded_gotoh(31, 1, (2, -2, -5, -3), *pr)
    assert same(run(31, 1, (2, -2, -5, -3), pr, pbits=4, tbits=2, tbe=True, max_m=160), want)
    # empty batch and a single alignment
    e = (np.zeros(4, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(4, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    s, x, y = run(31, 1, (2, -2, -5, -3), e, pbits=2, tbits=2, tbe=True)
    assert len(s) == 0
    one = fixed_problems(rng, 1, 31, 150)
    assert same(run(31, 1, (2, -2, -5, -3), one, pbits=2, tbits=2, tbe=True), O.banded_gotoh(31, 1, (2, -2, -5, -3), *one))
    # text shorter than the pattern -> BestSink defaults
    short = (np.zeros(10, np.uint8), np.array([0], np.uint32), np.array([10], np.uint32), np.zeros(8, np.uint8), np.array([0], np.uint32), np.array([5], np.uint32))
    s, x, y = run(31, 1, (2, -2, -5, -3), short, pbits=2, tbits=2, tbe=True)
    assert int(s[0]) == -2**30 and int(x[0]) == 0xFFFFFFFF            # NVB_SINK_MIN = the reference's Field_traits<int32>::min() and int(y[0]) == 0xFFFFFFFF


def test_quality_table_scheme(O):
    """nvBowtie's quality-dependent substitution (scoring.h:86-105,281) through the table interface"""
    rng = np.random.default_rng(4)
    pr = random_problems(rng, 2000, 31, 150, alphabet_text=5)
    qual = rng.integers(0, 60, len(pr[0])).astype(np.uint8)
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    assert sch.pgo == -8 and sch.pge == -3
    # the padded per-string quality layout: quals are indexed like the pattern stream
    for typ in (1, 2):
        want = O.banded_gotoh(31, typ, (2, int(sch.table_host[0, 1]), sch.pgo, sch.pge, sch.tgo, sch.tge), *pr, qual=qual, qtab=sch.table_host)
        assert same(run(31, typ, sch, pr, pbits=4, tbits=8, quals=qual), want)
    # nvBowtie-shaped jobs (2-bit genome windows, 4-bit reads): the packed DPX path builds its per-row profiles from the table
    for band in (15, 31):
        for typ in (1, 2):
            pr2 = fixed_problems(rng, 2001, band, 150, ragged=(typ == 1))
            qual2 = rng.integers(0, 60, len(pr2[0])).astype(np.uint8)
            want = O.banded_gotoh(band, typ, (2, int(sch.table_host[0, 1]), sch.pgo, sch.pge, sch.tgo, sch.tge), *pr2, qual=qual2, qtab=sch.table_host)
            force_path(0)
            for pbe in (True, False):
                assert same(run(band, typ, sch, pr2, pbits=4, tbits=2, pbe=pbe, tbe=True, quals=qual2, max_m=150), want), (band, typ, pbe)
            force_path(1)
            try:
                assert same(run(band, typ, sch, pr2, pbits=4, tbits=2, tbe=True, quals=qual2, max_m=150), want)
            finally:
                force_path(0)


def test_c1_sw_benchmark_banded(O):
    """BASELINE.json configs[0], banded variant (SURVEY 8d C1-ii): 10K x 100 bp patterns sampled from a 1 Kbp reference
    with 2% substitutions + 0.5% indels, BAND_LEN 15, GLOBAL, SimpleGotohScheme(2,-1,-2,-1) (sw-benchmark.cu:594-598),
    each against its 114 bp true window"""
    rng = np.random.default_rng(2024)
    ref = rng.integers(0, 4, 1000).astype(np.uint8)
    pats, p_off, p_len, t_off, t_len = [], [], [], [], []
    po = 0
    for _ in range(10000):
        st = int(rng.integers(0, 1000 - 114))
        j, p = st, []
        while len(p) < 100:
            r = rng.random()
            if r < 0.0025:
                p.append(int(rng.integers(0, 4)))            # insertion
            elif r < 0.005:
                j += 1                                        # deletion
            elif r < 0.025:
                p.append(int((ref[min(j, 999)] + 1 + rng.integers(0, 3)) % 4)); j += 1
            else:
                p.append(int(ref[min(j, 999)])); j += 1
        pats.append(np.array(p, np.uint8)); p_off.append(po); p_len.append(100); po += 100
        t_off.append(st); t_len.append(114)
    pr = (np.concatenate(pats), np.array(p_off, np.uint32), np.array(p_len, np.uint32), ref, np.array(t_off, np.uint32), np.array(t_len, np.uint32))
    for typ in (0, 2, 1):
        want = O.banded_gotoh(15, typ, (2, -1, -2, -1), *pr)
        assert same(run(15, typ, (2, -1, -2, -1), pr, pbits=4, tbits=2, tbe=False, max_m=100), want), typ


def test_scores_out_of_int16_budget_use_int32(O):
    """a scheme the packed path must refuse is still scored exactly (generic int32 kernel)"""
    rng = np.random.default_rng(8)
    pr = fixed_problems(rng, 500, 31, 150)
    for scheme in ((300, -200, -500, -300), (40, -2, -5, -3)):
        want = O.banded_gotoh(31, 1, scheme, *pr)
        assert same(run(31, 1, scheme, pr, pbits=2, tbits=2, tbe=True), want)


def test_full_size_properties():
    """C4-shaped batch (1M x 151 bp vs 300 bp windows): packed path == generic path bit for bit, scores of
    exact substrings equal 2*len, and results are invariant under batch permutation."""
    require_gpu()
    from nvbio_b200 import synth
    n_g, n, L, W = 4_000_000, 1_000_000, 151, 300
    gw = synth.random_genome_words(n_g)
    rw, pos, strand = synth.sample_reads(gw, n_g, n, L, rc_half=False)
    begin = synth.windows_for_reads(n_g, pos, L, W)
    P = PackedStringSet.fixed(rw.reshape(-1), n, L, stride=rw.shape[1] * 16)
    T = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=begin.to(torch.int32), lengths=None, stride=0, length=W, count=n)
    al = aln.make_gotoh_aligner(aln.LOCAL, aln.SimpleGotohScheme(2, -2, -5, -3))
    for band in (15, 31):
        force_path(0)
        s0, k0 = aln.batch_banded_alignment_score(band, al, P, T)
        force_path(1)
        try:
            s1, k1 = aln.batch_banded_alignment_score(band, al, P, T)
        finally:
            force_path(0)
        assert torch.equal(s0, s1) and torch.equal(k0, k1)
        assert int(s0.max()) <= 2 * L and int(s0.min()) >= 0
    # reads that are exact substrings score 2*L when the window offset is inside the band
    rw2, pos2, _ = synth.sample_reads(gw, n_g, 10000, L, sub_rate=0.0, indel_rate=0.0, rc_half=False)
    P2 = PackedStringSet.fixed(rw2.reshape(-1), 10000, L, stride=rw2.shape[1] * 16)
    T2 = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=(pos2 - 7).clamp_(0).to(torch.int32), lengths=None, stride=0, length=W, count=10000)
    s2, k2 = aln.batch_banded_alignment_score(31, al, P2, T2)
    assert bool((s2 == 2 * L).all())
    perm = torch.randperm(10000, device="cuda")
    T3 = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=T2.offsets[perm].contiguous(), lengths=None, stride=0, length=W, count=10000)
    P3 = PackedStringSet(words=P2.words, bits=2, big_endian=True, offsets=(perm * P2.stride).to(torch.int32), lengths=None, stride=0, length=L, count=10000)
    s3, k3 = aln.batch_banded_alignment_score(31, al, P3, T3)
    assert torch.equal(s3, s2[perm]) and torch.equal(k3, k2[perm])


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_full_matrix_score_vs_oracle(O, typ):
    """nvb_gotoh_score (full DP, SURVEY 8f-3) == the oracle (pinned against aln::alignment_score): scores, sinks, LOCAL tie order;
    ragged lengths from 1 symbol to several 32-column stripes, 2/4/8-bit packings"""
    from tests.test_host_core import full_problems
    rng = np.random.default_rng(900 + typ)
    for scheme in ((2, -1, -2, -1), (2, -2, -5, -3), (0, -5, -8, -3)):
        pr = full_problems(rng, 700, max_m=200, max_n=500)
        want = O.gotoh_full(typ, scheme, *pr)
        pat, p_off, p_len, txt, t_off, t_len = pr
        for pbits, tbits, tbe in ((4, 2, True), (2, 8, False)):
            P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits, big_endian=True)
            T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=tbits, big_endian=tbe)
            s, k = aln.batch_alignment_score(aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme)), P, T)
            torch.cuda.synchronize()
            k = host_u32(k)
            assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), (typ, scheme, pbits, tbits)


def test_full_matrix_reference_strings(O):
    p, t = orc.dna(G1_P), orc.dna(G1_T)
    for typ, want in ((0, (1, 20, 7)), (1, (13, 18, 7)), (2, (13, 18, 7))):
        P = PackedStringSet.from_symbols(p, [0], [len(p)], bits=2, big_endian=True)
        T = PackedStringSet.from_symbols(t, [0], [len(t)], bits=2, big_endian=True)
        s, k = aln.batch_alignment_score(aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -1, -1, -1)), P, T)
        k = host_u32(k)
        assert (int(s[0]), int(k[0, 0]), int(k[0, 1])) == want


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_full_matrix_packed_path(O, typ):
    """gotoh_full_pair_kernel (two alignments per thread, s16x2): consecutive alignments of equal shape take the packed path, the
    rest (ragged neighbours, N in the pattern) its int32 fallback; all == oracle; forcing the int32 kernel gives the same"""
    from tests.test_host_core import paired_full_problems
    rng = np.random.default_rng(950 + typ)
    for scheme in ((2, -1, -2, -1), (2, -2, -5, -3)):
        for n_frac in (0.0, 0.1):
            pr = paired_full_problems(rng, 600, max_m=200, max_n=400, n_frac=n_frac)
            want = O.gotoh_full(typ, scheme, *pr)
            pat, p_off, p_len, txt, t_off, t_len = pr
            P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
            T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
            al = aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme))
            nb.lib().nvb_debug_full_warp(C.c_int(2))           # thread-per-pair kernel at its three occupancy variants
            for minb in (2, 3, 4):
                nb.lib().nvb_debug_full_minb(C.c_int(minb))
                s, k = aln.batch_alignment_score(al, P, T)
                k = host_u32(k)
                assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), (typ, scheme, n_frac, minb)
            nb.lib().nvb_debug_full_minb(C.c_int(0))
            nb.lib().nvb_debug_full_warp(C.c_int(1))           # warp-per-pair wavefront kernel
            s, k = aln.batch_alignment_score(al, P, T)
            k = host_u32(k)
            nb.lib().nvb_debug_full_warp(C.c_int(0))
            assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), (typ, scheme, n_frac, "warp")
            force_path(1)
            try:
                s, k = aln.batch_alignment_score(al, P, T)
            finally:
                force_path(0)
            k = host_u32(k)
            assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), (typ, scheme, "int32")


def test_full_matrix_golden_gpu():
    """nvb_gotoh_score / nvb_gotoh_traceback == the committed outputs of the reference itself (tests/golden/gotoh_full.npz):
    score, sink, source, op stream; the reference-asserted 4M1D3M CIGAR of alignment_test.cu:784-793"""
    require_gpu()
    g = np.load(os.path.join(GOLD, "gotoh_full.npz"))
    p, t = orc.dna(G1_P), orc.dna(G1_T)
    for typ, cig in ((0, "1M2D3M1D3M10D"), (1, "4M1D3M"), (2, "4M1D3M")):
        P = PackedStringSet.from_symbols(p, [0], [len(p)], bits=2, big_endian=True)
        T = PackedStringSet.from_symbols(t, [0], [len(t)], bits=2, big_endian=True)
        tb = aln.batch_alignment_traceback(aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -1, -1, -1)), P, T)
        want = g[f"g1_t{typ}"]
        got = [int(tb["score"][0])] + [int(v) for v in host_u32(tb["sink"])[0]] + [int(v) for v in host_u32(tb["source"])[0]]
        assert got == [int(v) for v in want], (typ, got)
        # the reference's test strings are the backtracer's pushes in END -> START order (TestBacktracker, alignment_test_utils.h:628-643)
        assert orc.rle(tb["ops"][0].cpu().numpy()[:int(tb["n_ops"][0])]) == cig
    for cid, typ, m, mm, go, ge in g["cases"]:
        pr = [g[f"f{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len")]
        res, ops = g[f"f{cid}_res"], g[f"f{cid}_ops"]
        pat, p_off, p_len, txt, t_off, t_len = pr
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=2, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
        al = aln.make_gotoh_aligner(int(typ), aln.SimpleGotohScheme(int(m), int(mm), int(go), int(ge)))
        s, k = aln.batch_alignment_score(al, P, T)
        k = host_u32(k)
        assert np.array_equal(s.cpu().numpy().astype(np.int64), res[0]) and np.array_equal(k[:, 0].astype(np.int64), res[1]) and np.array_equal(k[:, 1].astype(np.int64), res[2]), cid
        tb = aln.batch_alignment_traceback(al, P, T, max_ops=512)
        src = host_u32(tb["source"]); n_ops = tb["n_ops"].cpu().numpy(); o = tb["ops"].cpu().numpy()
        assert np.array_equal(tb["score"].cpu().numpy().astype(np.int64), res[0]) and np.array_equal(host_u32(tb["sink"])[:, 0].astype(np.int64), res[1])
        assert np.array_equal(src[:, 0].astype(np.int64), res[3]) and np.array_equal(src[:, 1].astype(np.int64), res[4]) and np.array_equal(n_ops.astype(np.int64), res[5]), cid
        assert np.array_equal(np.concatenate([o[i][:n_ops[i]] for i in range(len(n_ops))]), ops), cid


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_full_matrix_traceback_vs_oracle(O, typ):
    from tests.test_host_core import full_problems
    rng = np.random.default_rng(990 + typ)
    for scheme in ((2, -1, -2, -1), (2, -2, -5, -3)):
        pr = full_problems(rng, 400, max_m=180, max_n=420)
        want = O.gotoh_full_traceback(typ, scheme, *pr, max_ops=640)
        pat, p_off, p_len, txt, t_off, t_len = pr
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
        tb = aln.batch_alignment_traceback(aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme)), P, T, max_ops=640)
        n_ops = tb["n_ops"].cpu().numpy(); o = tb["ops"].cpu().numpy()
        assert np.array_equal(tb["score"].cpu().numpy(), want["score"]) and np.array_equal(host_u32(tb["sink"]), want["sink"])
        assert np.array_equal(host_u32(tb["source"]), want["source"]) and np.array_equal(n_ops.astype(np.uint32), want["n_ops"])
        for i in range(len(n_ops)):
            assert np.array_equal(o[i][:n_ops[i]], want["ops"][i][:n_ops[i]]), (typ, scheme, i)


@pytest.mark.parametrize("band", [7, 15, 31])
def test_windowed_banded_score(O, band):
    """nvb_banded_gotoh_score_window: pass-by-pass state (BestSink, checkpoint bands, alive flags) == the oracle, and scoring in
    windows == nvb_banded_gotoh_score"""
    from tests.golden.make_golden import random_problems
    rng = np.random.default_rng(1200 + band)
    for typ in (0, 1, 2):
        scheme = (2, -2, -5, -3)
        pr = random_problems(rng, 500, band, 140, alphabet_text=6)
        pat, p_off, p_len, txt, t_off, t_len = pr
        n = len(p_off)
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=8, big_endian=False)
        al = aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme))
        whole = run(band, typ, scheme, pr)
        for W, ms in ((32, None), (32, rng.integers(-60, 140, n).astype(np.int32))):
            so = orc.window_state(n, band)
            st = aln.BandedWindowState(n, band, "cuda")
            msd = torch.from_numpy(ms).cuda() if ms is not None else None
            for wb in range(0, 140, W):
                O.banded_gotoh_window(band, typ, scheme, *pr, wb, wb + W, so, min_score=ms)
                aln.batch_banded_alignment_score_window(band, al, P, T, wb, wb + W, st, min_score=msd)
                torch.cuda.synchronize()
                k = host_u32(st.sink)
                assert np.array_equal(st.alive.cpu().numpy(), so["alive"]), (band, typ, wb)
                assert np.array_equal(st.score.cpu().numpy(), so["score"]) and np.array_equal(k[:, 0], so["sx"]) and np.array_equal(k[:, 1], so["sy"]), (band, typ, wb)
                alive = so["alive"].astype(bool)
                assert np.array_equal(st.ckpt.cpu().numpy()[alive], so["ckpt"][alive]), (band, typ, wb)
            if ms is None:
                ok = so["alive"].astype(bool)
                k = host_u32(st.sink)
                assert np.array_equal(st.score.cpu().numpy()[ok], whole[0][ok]) and np.array_equal(k[ok, 0], whole[1][ok]) and np.array_equal(k[ok, 1], whole[2][ok])


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_full_matrix_warp_kernel_every_width(O, typ):
    """gotoh_full_warp_kernel<TYPE, W> for every W = 1..8 (pattern lengths 1..256, incl. lengths that leave the last lane partly
    empty and put an 8-column stripe boundary inside a lane), short and long texts (fewer rows than lanes), LOCAL tie order"""
    from tests.test_host_core import paired_full_problems
    rng = np.random.default_rng(1300 + typ)
    nb.lib().nvb_debug_full_warp(C.c_int(1))
    try:
        for max_m in (7, 32, 33, 64, 90, 128, 150, 161, 200, 224, 256):
            for scheme in ((2, -1, -2, -1), (2, -2, -5, -3)):
                pr = paired_full_problems(rng, 150, max_m=max_m, max_n=330)
                want = O.gotoh_full(typ, scheme, *pr)
                pat, p_off, p_len, txt, t_off, t_len = pr
                P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=2, big_endian=True)
                P.length = max_m
                T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
                s, k = aln.batch_alignment_score(aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme)), P, T)
                k = host_u32(k)
                assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), (typ, max_m, scheme)
    finally:
        nb.lib().nvb_debug_full_warp(C.c_int(0))


def test_full_matrix_quality_table(O):
    """nvb_gotoh_score / nvb_gotoh_traceback with nvBowtie's quality-dependent scheme (QualityGotohScheme -> 256 x 2 table): scores and
    sinks == the oracle (pinned against the reference templates with a table-driven scheme); the traceback's score / sink agree"""
    from tests.test_host_core import full_problems, paired_full_problems
    rng = np.random.default_rng(1400)
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    tup = (2, int(sch.table_host[0, 1]), sch.pgo, sch.pge, sch.tgo, sch.tge)
    for typ in (0, 1, 2):
        for pr in (full_problems(rng, 400, max_m=160, max_n=400), paired_full_problems(rng, 200, max_m=160, max_n=300)):
            pat, p_off, p_len, txt, t_off, t_len = pr
            qual = rng.integers(0, 60, len(pat)).astype(np.uint8)
            want = O.gotoh_full(typ, tup, *pr, qual=qual, qtab=sch.table_host)
            P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
            T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
            q = torch.from_numpy(qual).cuda()
            al = aln.make_gotoh_aligner(typ, sch)
            s, k = aln.batch_alignment_score(al, P, T, quals=q)
            k = host_u32(k)
            assert same((s.cpu().numpy(), k[:, 0], k[:, 1]), want), typ
            tb = aln.batch_alignment_traceback(al, P, T, max_ops=600, quals=q)
            assert np.array_equal(tb["score"].cpu().numpy(), want[0]) and np.array_equal(host_u32(tb["sink"])[:, 0], want[1])


def test_windowed_and_quality_golden_gpu():
    """nvb_banded_gotoh_score_window and the quality-table paths of nvb_banded_gotoh_score / nvb_gotoh_score == the committed
    outputs of the reference itself (tests/golden/banded_extras.npz)"""
    require_gpu()
    g = np.load(os.path.join(GOLD, "banded_extras.npz"))
    for cid, band, typ in g["wcases"]:
        band, typ = int(band), int(typ)
        pat, p_off, p_len, txt, t_off, t_len = [g[f"w{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len")]
        ms = g[f"w{cid}_ms"]
        n = len(p_off)
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=8, big_endian=False)
        al = aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -2, -5, -3))
        st = aln.BandedWindowState(n, band, "cuda")
        msd = torch.from_numpy(ms).cuda() if len(ms) else None
        for w, wb in enumerate(range(0, 100, 32)):
            aln.batch_banded_alignment_score_window(band, al, P, T, wb, wb + 32, st, min_score=msd)
            k = host_u32(st.sink)
            snap = np.concatenate([st.score.cpu().numpy().astype(np.int64), k[:, 0].astype(np.int64), k[:, 1].astype(np.int64), st.alive.cpu().numpy().astype(np.int64)])
            assert np.array_equal(snap, g[f"w{cid}_snaps"][w]), (cid, band, typ, wb)
        alive = st.alive.cpu().numpy().astype(bool)
        assert np.array_equal(st.ckpt.cpu().numpy()[alive], g[f"w{cid}_ckpt"][alive]), cid

    class _TableScheme:                       # the fixture's table behind the scheme interface of nvbio_b200.aln
        def __init__(self, tab):
            self.table_host = np.ascontiguousarray(tab); self.table = torch.from_numpy(self.table_host).cuda()

        def struct(self):
            from nvbio_b200._lib import GotohSchemeStruct
            s = GotohSchemeStruct()
            s.match, s.mismatch, s.pattern_gap_open, s.pattern_gap_ext, s.text_gap_open, s.text_gap_ext = 0, 0, -8, -3, -7, -2
            s.d_qual_table = self.table.data_ptr(); s.qual_table_min, s.qual_table_max = int(self.table_host.min()), int(self.table_host.max())
            return s
    sch = _TableScheme(g["qtab"])
    for cid, band, typ in g["qcases"]:
        band, typ = int(band), int(typ)
        pat, p_off, p_len, txt, t_off, t_len = [g[f"q{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len")]
        qual, res = g[f"q{cid}_qual"], g[f"q{cid}_res"]
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2 if not band else 8, big_endian=bool(not band))
        q = torch.from_numpy(qual).cuda()
        al = aln.make_gotoh_aligner(typ, sch)
        if band:
            s, k = aln.batch_banded_alignment_score(band, al, P, T, quals=q)
        else:
            s, k = aln.batch_alignment_score(al, P, T, quals=q)
        k = host_u32(k)
        ok = res[3].astype(bool)
        assert np.array_equal(s.cpu().numpy().astype(np.int64)[ok], res[0][ok]), (cid, band, typ)
        assert np.array_equal(k[:, 0].astype(np.int64)[ok], res[1][ok]) and np.array_equal(k[:, 1].astype(np.int64)[ok], res[2][ok]), (cid, band, typ)


def test_quality_scheme_vs_nvbowtie_scheme_object():
    """nvb_banded_gotoh_score with nvbio_b200.aln.QualityGotohScheme(--local constants) == aln::banded_alignment_score run with
    nvBowtie's OWN scheme object SmithWatermanScoringScheme<QualCost<int>,ConstantCost<int>>::local() and per-base qualities
    (committed outputs of the reference: tests/golden/nvbowtie_scheme.npz, make_golden.py make_nvbowtie); LOCAL + SEMI_GLOBAL, bands 15 / 31"""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "nvbowtie_scheme.npz"))
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    assert np.array_equal(sch.table_host, g["tab0"])
    for cid, band, typ in g["dcases"]:
        pr = [g[f"d{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len")]
        res = g[f"d{cid}_res"]
        ok = pr[5] >= pr[2]
        s, x, y = run(int(band), int(typ), sch, pr, pbits=4, tbits=8, quals=g[f"d{cid}_qual"])
        assert np.array_equal(np.asarray(s, np.int64)[ok], res[0][ok]) and np.array_equal(np.asarray(x, np.int64)[ok], res[1][ok]) \
            and np.array_equal(np.asarray(y, np.int64)[ok], res[2][ok]), (cid, band, typ)


def test_best2_sink(O):
    """nvb_banded_gotoh_score_best2 == the banded DP feeding aln::Best2Sink<int32>(distinct_dist) (oracle restatement, itself pinned to the
    reference templates in tests/test_oracle.py): best and distinct second-best (score, sink) of every alignment"""
    rng = np.random.default_rng(8)
    for band in (7, 15, 31):
        for typ in (0, 1, 2):
            for dist in (0, 10):
                pr = random_problems(rng, 500, band, 150)
                pat, p_off, p_len, txt, t_off, t_len = pr
                P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
                T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=8, big_endian=False)
                got = aln.batch_banded_alignment_score_best2(band, aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -2, -5, -3)), P, T, distinct_dist=dist)
                torch.cuda.synchronize()
                want = O.banded_gotoh_best2(band, typ, (2, -2, -5, -3), *pr, distinct_dist=dist)
                g = got.cpu().numpy().astype(np.int64)
                g[:, [1, 2, 4, 5]] &= 0xFFFFFFFF
                valid = t_len >= p_len
                assert np.array_equal(g[valid], want[valid]), (band, typ, dist)
