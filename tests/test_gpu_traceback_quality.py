"""-m gpu: the Gotoh tracebacks under nvBowtie's quality-table scheme (QualityGotohScheme + per-base qualities) on the device == the oracle's
quality traceback (pinned to the reference's own templates by tests/test_traceback_quality_host.py): score, sink, source, n_ops and every op.

- nvb_banded_gotoh_traceback at bands 3 / 5 / 7 / 15 / 31, every type, through the gapless fast path and with every alignment through the
  direction matrix, 2- and 4-bit patterns with N's, every quality profile, match bonus 2 (LOCAL) and 0 (end-to-end), and at the packed
  score pass's selector cap;
- nvb_gotoh_traceback (the direction-matrix kernel and the warp traceback) at every warp-width boundary of M up to 512, N up to 1000;
- ops truncated at max_ops on every path: n_ops stays the full count, the stored prefix is the oracle's, nothing is written past it;
- seed_extend / seed_extend_paired with traceback=True: every read's ops and begin == the oracle's quality traceback of its best job, every
  rescued mate's == the oracle's full-matrix quality traceback of the winning opposite-mate job."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200._lib import lib, check
from nvbio_b200.strings import PackedStringSet, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import seed_extend_oracle, best_hits, _scheme_args
from tests.test_gpu_gotoh_limits import debug_knobs, last_route, assert_route, banded_batch
from tests.golden.make_traceback_quality_golden import banded_problems, full_problems, qualities, _mutate, _pack

GLOBAL, LOCAL, SEMI = aln.GLOBAL, aln.LOCAL, aln.SEMI_GLOBAL
SENT = 0xAB                       # what an op byte the device must not write keeps
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


def qscheme(mb):
    """nvBowtie's scheme with match bonus mb, mismatch 2..6 by quality, read gaps 5 + 3k, reference gaps 5 + 2k (text gaps cost less)"""
    return aln.QualityGotohScheme(mb, 2, 6, 5, 3, 5, 2)


def bonuses(typ):
    return (2,) if typ == LOCAL else (2, 0)


def device_traceback(band, typ, scheme, pr, qual, max_ops, pbits=4, tbits=4):
    """nvb_banded_gotoh_traceback (band > 0) / nvb_gotoh_traceback (band 0) with an op buffer prefilled with SENT and 64 bytes of slack"""
    pat, p_off, p_len, txt, t_off, t_len = pr
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits, big_endian=True)
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=tbits, big_endian=True)
    n = len(p_off)
    dev = P.words.device
    score = torch.empty(n, dtype=torch.int32, device=dev); sink = torch.empty((n, 2), dtype=torch.int32, device=dev)
    source = torch.empty((n, 2), dtype=torch.int32, device=dev); n_ops = torch.empty(n, dtype=torch.int32, device=dev)
    ops = torch.full((n * max_ops + 64,), SENT, dtype=torch.uint8, device=dev)
    q = torch.from_numpy(np.ascontiguousarray(qual)).cuda() if qual is not None else None
    sch, p, t = scheme.struct(), P.struct(), T.struct()
    qp = C.c_void_p(q.data_ptr()) if q is not None else None
    tb = C.c_size_t(0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    outs = [C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()), C.c_void_p(source.data_ptr()), C.c_void_p(ops.data_ptr()),
            C.c_uint32(max_ops), C.c_void_p(n_ops.data_ptr())]

    def call(temp):
        if band:
            return lib().nvb_banded_gotoh_traceback(C.c_int(band), C.c_int(typ), C.byref(sch), C.byref(p), qp, C.byref(t), C.c_uint32(n),
                                                    *outs, temp, C.byref(tb), stream)
        return lib().nvb_gotoh_traceback(C.c_int(typ), C.byref(sch), C.byref(p), qp, C.byref(t), C.c_uint32(n), *outs, temp, C.byref(tb), stream)
    r = call(None)
    if r != -2:
        check(r, "traceback (size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(call(C.c_void_p(temp.data_ptr())), "traceback")
    torch.cuda.synchronize()
    flat = ops.cpu().numpy()
    return dict(score=score.cpu().numpy(), sink=host_u32(sink), source=host_u32(source), n_ops=n_ops.cpu().numpy().astype(np.uint32),
                ops=flat[:n * max_ops].reshape(n, max_ops), slack=flat[n * max_ops:])


def oracle_traceback(O, band, typ, scheme, pr, qual, max_ops):
    s6, qtab = _scheme_args(scheme)
    if band:
        return O.banded_traceback(band, typ, s6, *pr, max_ops=max_ops, qual=qual if qtab is not None else None, qtab=qtab)
    return O.gotoh_full_traceback(typ, s6, *pr, max_ops=max_ops, qual=qual if qtab is not None else None, qtab=qtab)


def assert_traceback(got, want, max_ops, what):
    """score, sink, source and n_ops (the full count) == the oracle's; the first min(n_ops, max_ops) bytes of every row are the oracle's
    ops, the rest of the row and the slack behind the last row keep SENT"""
    for k in ("score", "sink", "source", "n_ops"):
        g, w = np.asarray(got[k]).astype(np.int64), np.asarray(want[k]).astype(np.int64)
        bad = np.flatnonzero((g != w).reshape(len(g), -1).any(axis=1))
        assert len(bad) == 0, "%s: %s differs at %d alignments, first %d: got %s want %s" % (what, k, len(bad), bad[0], g[bad[0]], w[bad[0]])
    for i in range(len(got["n_ops"])):
        k = min(int(got["n_ops"][i]), max_ops)
        assert np.array_equal(got["ops"][i, :k], want["ops"][i, :k]), (what, i)
        assert (got["ops"][i, k:] == SENT).all(), (what, i, "written past the ops")
    assert (got["slack"] == SENT).all(), (what, "written past the last row")


def gapless_count(want, pr):
    """alignments whose traceback is all substitutions with no N in pattern or window: those the gapless fast path claims (its claim set
    is exactly these, tests/test_traceback_quality_host.py::test_host_gapless_fast_path_quality)"""
    pat, p_off, p_len, txt, t_off, t_len = pr
    c = 0
    for a in range(len(p_off)):
        k = int(want["n_ops"][a])
        c += int(k > 0 and not want["ops"][a][:k].any() and not (pat[p_off[a]:p_off[a] + p_len[a]] > 3).any()
                 and not (txt[t_off[a]:t_off[a] + t_len[a]] > 3).any())
    return c


# --------------------------------------------------------------------------------------------------------------------------------------
# banded
# --------------------------------------------------------------------------------------------------------------------------------------
BANDED_BATCHES = (   # (name, generator keywords, pattern bits, text bits)
    ("gapless-low", dict(indel=0.002, sub=0.02, profile="low"), 2, 2),
    ("gapless-high", dict(indel=0.002, sub=0.03, profile="high"), 2, 2),
    ("gapless-clamp", dict(indel=0.002, sub=0.02, profile="clamp", ragged=False), 2, 2),
    ("gap-rich", dict(indel=0.02, tie=1.0, profile="rand"), 2, 2),
    ("N", dict(n_pat=0.02, n_txt=0.01, profile="rand"), 4, 4),
    ("N-pattern", dict(n_pat=0.02, indel=0.01, profile="mixed"), 4, 2),
)


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
@pytest.mark.parametrize("band", [3, 5, 7, 15, 31])
def test_banded_quality_traceback(O, band, typ):
    require_gpu()
    rng = np.random.default_rng(5000 + 10 * band + typ)
    for mb in bonuses(typ):
        scheme = qscheme(mb)
        for name, kw, pbits, tbits in BANDED_BATCHES:
            pr, qual = banded_problems(rng, 301, band, 150, **kw)
            max_ops = 2 * 150 + band
            want = oracle_traceback(O, band, typ, scheme, pr, qual, max_ops)
            if name.startswith("gapless") and typ != GLOBAL:
                assert gapless_count(want, pr) > 0.5 * len(pr[1]), (band, typ, mb, name)
            for fast in (1, 0):
                with debug_knobs(traceback_fast=fast):
                    got = device_traceback(band, typ, scheme, pr, qual, max_ops, pbits, tbits)
                assert_traceback(got, want, max_ops, "B%d t%d mb%d %s fast=%d" % (band, typ, mb, name, fast))


@pytest.mark.gpu
@pytest.mark.parametrize("band", [7, 15, 31])
def test_banded_quality_traceback_at_the_selector_cap(O, band):
    """the longest patterns the packed score pass admits (and one longer) under a quality table, through the fast path and the direction
    matrix; the fast path's score pass is the packed kernel exactly when the selector rows fit"""
    require_gpu()
    cap = 801 - band
    for m in (cap, cap + 1):
        rng = np.random.default_rng(band * 1000 + m + 7)
        pr = banded_batch(rng, band, m, n=31)
        qual = qualities(rng, len(pr[0]), "rand")
        max_ops = m + band + 1
        for typ in (GLOBAL, LOCAL, SEMI):
            scheme = qscheme(2 if typ == LOCAL else 0)
            want = oracle_traceback(O, band, typ, scheme, pr, qual, max_ops)
            for fast in (1, 0):
                with debug_knobs(traceback_fast=fast):
                    got = device_traceback(band, typ, scheme, pr, qual, max_ops, 4, 2)
                    route = last_route()
                what = "B%d m%d t%d fast=%d" % (band, m, typ, fast)
                assert_traceback(got, want, max_ops, what)
                assert_route(route, fast == 1 and typ != GLOBAL and m == cap, what)


# --------------------------------------------------------------------------------------------------------------------------------------
# full matrix
# --------------------------------------------------------------------------------------------------------------------------------------
def warp_width_problems(rng, max_n=1000, per=2):
    """per problems at every M = 32 k and 32 k + 1 (every lane width W = ceil(M / 32) of the warp traceback and both sides of each
    boundary) up to 512, texts of up to max_n symbols, mostly drawn from their text with indels and low-quality mismatches beside them"""
    items = []
    for M in [1, 2] + [v for k in range(1, 16) for v in (32 * k, 32 * k + 1)] + [511, 512]:
        for _ in range(per):
            N = int(rng.integers(max(1, M // 2), max_n + 1))
            t = rng.integers(0, 4, N).astype(np.uint8)
            if N > M + 2 and rng.random() < 0.85:
                p, low = _mutate(rng, t, int(rng.integers(0, N - M - 1)), M, 0.015, 0.03, 0.5)
            else:
                p, low = rng.integers(0, 4, M).astype(np.uint8), np.zeros(M, bool)
            q = qualities(rng, M, "mixed")
            q[low] = rng.integers(0, 12, int(low.sum()))
            items.append((p, q, t))
    return _pack(items)


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
def test_full_quality_traceback(O, typ):
    """nvb_gotoh_traceback with a table: the direction-matrix kernel and the warp traceback (nvb_debug_full_traceback_warp(1)), both
    against the oracle"""
    require_gpu()
    rng = np.random.default_rng(5100 + typ)
    for mb in bonuses(typ):
        scheme = qscheme(mb)
        for pr, qual in (warp_width_problems(rng), full_problems(rng, 40, 512, 1000, n_pat=0.02, profile="low")):
            max_ops = int(pr[2].max()) + int(pr[5].max()) + 1
            want = oracle_traceback(O, 0, typ, scheme, pr, qual, max_ops)
            for warp in (0, 1):
                with debug_knobs(full_traceback_warp=warp):
                    got = device_traceback(0, typ, scheme, pr, qual, max_ops, 4, 2)
                assert_traceback(got, want, max_ops, "t%d mb%d warp=%d" % (typ, mb, warp))


# --------------------------------------------------------------------------------------------------------------------------------------
# truncation
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("scheme_kind", ["simple", "quality"])
def test_traceback_truncated_at_max_ops(O, scheme_kind):
    """max_ops in {1, K - 1, K // 2} (K the longest op count of the batch; fixed-length gapless batches: every row's count): n_ops is the
    full count, the stored prefix the oracle's, nothing written past max_ops -- the gapless fast path, the direction-matrix banded
    traceback, the full-matrix kernel and the warp traceback"""
    require_gpu()
    rng = np.random.default_rng(5200 + (scheme_kind == "quality"))
    for typ in (GLOBAL, LOCAL, SEMI):
        scheme = aln.SimpleGotohScheme(2, -6, -8, -3) if scheme_kind == "simple" else qscheme(2 if typ == LOCAL else 0)
        paths = [(31, "fast", dict(traceback_fast=1), banded_problems(rng, 97, 31, 120, indel=0.002, sub=0.02, ragged=False)),
                 (15, "dirs", dict(traceback_fast=0), banded_problems(rng, 97, 15, 150, indel=0.02)),
                 (0, "full", dict(full_traceback_warp=0), full_problems(rng, 33, 200, 400)),
                 (0, "warp", dict(full_traceback_warp=1), full_problems(rng, 33, 200, 400))]
        for band, name, knobs, (pr, qual) in paths:
            full = oracle_traceback(O, band, typ, scheme, pr, qual, 1200)
            K = int(full["n_ops"].max())
            for max_ops in sorted({1, K - 1, K // 2}):
                want = oracle_traceback(O, band, typ, scheme, pr, qual, max_ops)
                assert np.array_equal(want["n_ops"], full["n_ops"])
                with debug_knobs(**knobs):
                    got = device_traceback(band, typ, scheme, pr, qual, max_ops, 4, 2)
                what = "%s t%d %s max_ops=%d" % (scheme_kind, typ, name, max_ops)
                assert_traceback(got, want, max_ops, what)
                assert (got["n_ops"] > max_ops).any(), what                       # something was truncated
                if name == "fast" and typ != GLOBAL:
                    assert gapless_count(full, pr) > 0.5 * len(pr[1]), what


# --------------------------------------------------------------------------------------------------------------------------------------
# through seed + extend
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def world():
    """300 kbp genome; 400 single reads of 100-150 bp away from the genome's ends (2 % substitutions, 1-2 % indels with low-quality
    mismatches beside some, either strand) and 300 pairs of 100 bp; base qualities of every profile"""
    require_gpu()
    O = orc.Oracle()
    n = 300_000
    gw = synth.random_genome_words(n, seed=91)
    gsym = unpack_symbols(host_u32(gw), n)
    idx = O.build_index(gsym)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    rng = np.random.default_rng(92)
    reads, quals = [], []
    for i in range(400):
        m = int(rng.integers(100, 151))
        st = int(rng.integers(1000, n - 1000))
        r, low = _mutate(rng, gsym[st:st + m + 40], 0, m, [0.0, 0.01, 0.02][i % 3], 0.02, 0.7)
        q = qualities(rng, m, ("low", "high", "rand", "clamp", "mixed")[i % 5])
        q[low] = rng.integers(0, 12, int(low.sum()))
        if rng.random() < 0.5:
            r, q = np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8), q[::-1].copy()
        reads.append(r); quals.append(q)
    n_pairs = 300
    rw, _, _ = synth.sample_pairs(gw, n, n_pairs, 100, frag_mean=300, frag_sd=40, sub_rate=0.02, hard_frac=0.3, hard_sub_rate=0.2,
                                  seed=93, mut_seed=94)
    preads = [unpack_symbols(host_u32(rw[i]), 100).astype(np.uint8) for i in range(2 * n_pairs)]
    for i in rng.choice(2 * n_pairs, 120, replace=False):
        p, k = int(rng.integers(25, 75)), int(rng.integers(1, 4))
        r = preads[i]
        preads[i] = np.concatenate([r[:p], r[p + k:]]) if rng.random() < 0.5 else np.concatenate([r[:p], rng.integers(0, 4, k).astype(np.uint8), r[p:]])
    pquals = [qualities(rng, len(r), "rand") for r in preads]
    return dict(O=O, idx=idx, gsym=gsym, gw=gw, fmi=fmi, reads=reads, quals=quals, preads=preads, pquals=pquals, n_pairs=n_pairs)


def read_set(reads):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = (np.cumsum(lens) - lens).astype(np.uint32)
    return PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=2, big_endian=True)


def strand_string(r, q, strand):
    if strand == 0:
        return r, q
    return np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8), q[::-1]


def check_traceback(w, reads, quals, p, want, rows_got, what):
    """check_traceback of tests/test_gpu_pipeline_matrix.py with qualities: every read's ops and begin == the oracle's quality traceback of
    the read's best job (the reverse-complement strand with the reversed qualities).  rows_got[r] = (ops, n_ops, begin, strand) or None
    (a read the caller does not check); returns the number of reads checked"""
    scheme6, qtab = _scheme_args(p.scheme)
    bh = best_hits(want, len(reads))
    rows = [r for r in np.flatnonzero(bh >= 0) if rows_got[r] is not None]
    for r in np.flatnonzero(bh < 0):
        if rows_got[r] is not None:
            assert rows_got[r][1] == 0 and tuple(rows_got[r][2]) == (NONE, NONE), (what, r)
    pats, pq, t_off, t_len = [], [], [], []
    for r in rows:
        h = bh[r]
        s = int(want["hit_string"][h]) % 2
        pt, qt = strand_string(reads[r], quals[r], s)
        pats.append(pt); pq.append(qt)
        t_off.append(int(want["hit_window"][h][0])); t_len.append(int(want["hit_window"][h][1] - want["hit_window"][h][0]))
        assert rows_got[r][3] == s, (what, r)
    if not rows:
        return 0
    lens = np.array([len(x) for x in pats], np.uint32)
    max_ops = rows_got[rows[0]][0].shape[0]
    o = w["O"].banded_traceback(p.band_len, p.type, scheme6, np.concatenate(pats), (np.cumsum(lens) - lens).astype(np.uint32), lens,
                                w["gsym"], np.array(t_off, np.uint32), np.array(t_len, np.uint32), max_ops=max_ops,
                                qual=np.concatenate(pq), qtab=qtab)
    for a, r in enumerate(rows):
        ops, n_ops, begin, _ = rows_got[r]
        assert n_ops == o["n_ops"][a], (what, r)
        assert np.array_equal(ops[:min(n_ops, max_ops)], o["ops"][a, :min(n_ops, max_ops)]), (what, r)
        assert tuple(int(v) for v in begin) == (t_off[a] + int(o["source"][a][0]), int(o["source"][a][1])), (what, r)
    return len(rows)


def se_params(w, band, typ, quals):
    q = torch.from_numpy(np.concatenate(quals)).cuda()
    return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=band, type=typ, both_strands=True, max_seed_hits=50,
                               scheme=qscheme(2 if typ == LOCAL else 0), read_quals=q)


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
@pytest.mark.parametrize("band", [15, 31])
def test_seed_extend_quality_traceback(world, band, typ):
    w = world
    reads, quals = w["reads"], w["quals"]
    p = se_params(w, band, typ, quals)
    want = seed_extend_oracle(w["O"], w["idx"], w["gsym"], reads, p, quals=quals)
    cap = 2 * ((150 - 20) // 10 + 1) * p.max_seed_hits * len(reads) + 1024
    ws = nb.seed_extend(w["fmi"], w["gw"], read_set(reads), p, hit_capacity=cap, traceback=True)
    torch.cuda.synchronize()
    assert np.array_equal(ws.best_score.cpu().numpy().astype(np.int64), want["best_score"])
    ops, n_ops, begin, strand = ws.best_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy(), host_u32(ws.best_begin), ws.best_strand.cpu().numpy()
    got = [(ops[r], int(n_ops[r]), begin[r], int(strand[r])) for r in range(len(reads))]
    checked = check_traceback(w, reads, quals, p, want, got, (band, typ))
    assert checked > 0.9 * len(reads)
    assert len(set(int(v) for r in range(len(reads)) for v in ops[r, :n_ops[r]])) == 3          # M, I and D all occur


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
@pytest.mark.parametrize("band", [15, 31])
def test_seed_extend_paired_quality_traceback(world, band, typ):
    """mates aligned on their own == the oracle's banded quality traceback of their best job; rescued mates == the oracle's full-matrix
    quality traceback of the winning opposite-mate job (rebuilt from the anchor's oracle best hit by the rule of seed_extend_paired_oracle)"""
    w = world
    reads, quals, n_pairs = w["preads"], w["pquals"], w["n_pairs"]
    p = se_params(w, band, typ, quals)
    # end-to-end scores are <= 0: a rescued mate with a fifth of its bases mismatched (the hard mates) scores about -80
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50 if typ == LOCAL else -150)
    ws = nb.seed_extend_paired(w["fmi"], w["gw"], read_set(reads), p, pair, hit_capacity=64 * 2 * n_pairs, traceback=True)
    torch.cuda.synchronize()
    flags, mops, mn = ws.pair_flags.cpu().numpy(), ws.mate_ops.cpu().numpy(), ws.mate_n_ops.cpu().numpy()
    mbeg, mstrand = ws.mate_begin.cpu().numpy().view(np.uint32), ws.mate_strand.cpu().numpy()
    mscore, mpos = ws.mate_score.cpu().numpy(), ws.mate_pos.cpu().numpy().view(np.uint32)
    max_ops = ws.max_ops
    want = seed_extend_oracle(w["O"], w["idx"], w["gsym"], reads, p, quals=quals)
    rescued = [(q, 0 if flags[q] == 2 else 1) for q in range(n_pairs) if flags[q] in (2, 4)]
    rescued_set = set(rescued)
    got = [None] * (2 * n_pairs)
    for q in range(n_pairs):
        for m in range(2):
            if (q, m) not in rescued_set:
                got[m * n_pairs + q] = (mops[m, q], int(mn[m, q]), mbeg[m, q], int(mstrand[m, q]))
    check_traceback(w, reads, quals, p, want, got, (band, typ, "own"))
    # rescued mates
    bh = best_hits(want, len(reads))
    s6, qtab = _scheme_args(p.scheme)
    glen = w["idx"].n
    pats, pq, t_off, t_len = [], [], [], []
    for q, o in rescued:
        ra, ro = (1 - o) * n_pairs + q, o * n_pairs + q
        h = bh[ra]
        end = int(want["hit_window"][h][0] + want["hit_sink"][h][0]); beg = max(end - len(reads[ra]), 0)
        anchor_strand = int(want["hit_string"][h]) % 2
        to, te = (beg, min(beg + pair.max_frag, glen)) if anchor_strand == 0 else (max(end - pair.max_frag, 0), end)
        pt, qt = strand_string(reads[ro], quals[ro], 1 - anchor_strand)
        pats.append(pt); pq.append(qt); t_off.append(to); t_len.append(te - to)
    if typ != GLOBAL:
        assert len(rescued) > 0.05 * n_pairs, (band, typ, len(rescued))
    if rescued:
        lens = np.array([len(x) for x in pats], np.uint32)
        o = w["O"].gotoh_full_traceback(p.type, s6, np.concatenate(pats), (np.cumsum(lens) - lens).astype(np.uint32), lens, w["gsym"],
                                        np.array(t_off, np.uint32), np.array(t_len, np.uint32), max_ops=max_ops, qual=np.concatenate(pq), qtab=qtab)
        for i, (q, m) in enumerate(rescued):
            what = (band, typ, "rescued", q, m)
            assert mscore[m, q] == o["score"][i] and mpos[m, q] == t_off[i] + o["sink"][i][0], what
            assert mn[m, q] == o["n_ops"][i] and tuple(int(v) for v in mbeg[m, q]) == (t_off[i] + int(o["source"][i][0]), int(o["source"][i][1])), what
            k = min(int(mn[m, q]), max_ops)
            assert np.array_equal(mops[m, q, :k], o["ops"][i, :k]), what
