"""-m gpu: seed + extend against the oracle composition (tests/pipeline_oracle.py) across the parameter space the C ABI accepts, not only
at the headline point (band 31, LOCAL, one scheme, seeds longer than the k-mer table, reads inside the genome):

  a. every band (3, 5, 7, 15, 31, 63: the DPX pair kernel and the generic kernel) at LOCAL and every alignment type at bands 7, 15 and
     63, under five schemes -- one with zero gap extension and one whose pattern and text gaps differ -- hit by hit on the per-hit path,
     and per read on the per-read path with the exact shortcut on, without its one-gap check and off;
  b. seed geometry around a k = 10 k-mer table (seeds shorter than, equal to and longer than k, an interval wider than the seed, one hit
     per seed, 4-bit reads shorter than a seed) with the plain, located, context and per-row-array tables, in one and two passes;
  c. the best alignment's traceback at every band the traceback supports and every type, equal to the oracle's traceback of the read's
     best job, and band 63 refused by the traceback;
  d. paired end-to-end (SEMI_GLOBAL, no match bonus, nvBowtie's end-to-end --score-min) and LOCAL at band 15: pairs, paired MAPQ and both
     mates' alignments.

The genome (300,007 symbols: not a multiple of 16) has a period-7 tandem repeat and a period-300 repeat family; hand-placed reads start at
position 0, end at the genome's end, run past it by 1 to 70 symbols (a read more than band/2 past the end only gets windows shorter than
itself: the DP reports them empty and the read must come out unaligned), carry two substitutions (the shortcut's one-gap branch) or a
one-base indel a few rows from an end."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200._lib import GotohSchemeStruct, NvbError
from nvbio_b200.strings import PackedStringSet, pack_symbols, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import seed_extend_oracle, seed_extend_paired_oracle, best_hits, _scheme_args, EMPTY_SINK
from tests.pair_mapq_oracle import pair_mapq_oracle
from tests.test_gpu_paired_traceback import replay, strand_string, PAIR_KEYS, TB_KEYS, MAPQ_KEYS

pytestmark = pytest.mark.gpu

N_GENOME = 300_007
L = 150
INT_MIN = -2**31
NONE = 0xFFFFFFFF
OVERHANGS = (1, 2, 3, 4, 7, 8, 15, 16, 17, 31, 32, 33, 45, 70)       # every band/2 and band/2 + 1 of bands 3 .. 63


class AsymGotohScheme:
    """a scheme whose pattern and text gaps cost differently, through the C struct (SimpleGotohScheme has one gap cost)"""

    def __init__(self, match, mismatch, pgo, pge, tgo, tge):
        self.match, self.mismatch, self.pgo, self.pge, self.tgo, self.tge = match, mismatch, pgo, pge, tgo, tge

    def struct(self):
        s = GotohSchemeStruct()
        s.match, s.mismatch, s.pattern_gap_open, s.pattern_gap_ext, s.text_gap_open, s.text_gap_ext = \
            self.match, self.mismatch, self.pgo, self.pge, self.tgo, self.tge
        s.d_qual_table = None
        s.qual_table_min = s.qual_table_max = 0
        return s

    def __repr__(self):
        return "Asym(%d,%d,%d,%d,%d,%d)" % (self.match, self.mismatch, self.pgo, self.pge, self.tgo, self.tge)


SCHEMES = [aln.SimpleGotohScheme(2, -2, -5, -3), aln.SimpleGotohScheme(1, -4, -6, -1), aln.SimpleGotohScheme(3, -1, -2, -2),
           aln.SimpleGotohScheme(2, -3, -4, 0), AsymGotohScheme(2, -2, -5, -3, -9, -1)]
BAND_TYPES = [(b, aln.LOCAL) for b in (3, 5, 7, 15, 31, 63)] + [(b, t) for t in (aln.GLOBAL, aln.SEMI_GLOBAL) for b in (7, 15, 63)]


def _debug(name, v):
    getattr(nb.lib(), name)(C.c_int(v))


def rc(r):
    return np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8)


def hand_reads(g, n, rng):
    """reads at position 0 and at the genome's end, past the end by OVERHANGS symbols (random tail), each also reverse-complemented; two
    substitutions; a one-base deletion / insertion 3 to 6 rows from either end; reads inside the tandem repeat and the repeat family"""
    out = []
    for r in (g[:L], g[n - L:]):
        out += [r.copy(), rc(r)]
    for k in OVERHANGS:
        r = np.concatenate([g[n - L + k:], rng.integers(0, 4, k).astype(np.uint8)])
        out += [r, rc(r)]
    for p, q in ((30, 100), (10, 140), (74, 75), (40, 41), (16, 133), (60, 90)) * 3:
        st = int(rng.integers(200_000, n - 1000))
        r = g[st:st + L].copy()
        r[p] = (r[p] + 1) % 4; r[q] = (r[q] + 2) % 4
        out.append(r)
    for k in (3, 4, 5, 6):
        for at_end in (False, True):
            for insert in (False, True):
                st = int(rng.integers(160_000, n - 1000)); cut = L - k if at_end else k
                r = np.concatenate([g[st:st + cut], rng.integers(0, 4, 1).astype(np.uint8), g[st + cut:st + L - 1]]) if insert else \
                    np.concatenate([g[st:st + cut], g[st + cut + 1:st + L + 1]])
                out.append(r)
    for st in rng.integers(52_000, 68_000, 6):
        out.append(g[st:st + L].copy())
    for st in rng.integers(121_000, 148_000, 6):
        out.append(g[st:st + L].copy())
    return out


@pytest.fixture(scope="module")
def world():
    require_gpu()
    O = orc.Oracle()
    n = N_GENOME
    g = unpack_symbols(host_u32(synth.random_genome_words(n, seed=301)), n).copy()
    g[50_000:70_000] = np.tile(g[1000:1007], 20_000 // 7 + 1)[:20_000]
    g[120_000:150_000] = np.tile(g[2000:2300], 100)
    gw = torch.from_numpy(pack_symbols(np.concatenate([g, np.zeros(128, np.uint8)]), 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi, _ = nb.FMIndexDevice.from_text(gw, n, sa_interval=1)
    fmi.build_ktab(10, located=True, text=gw)
    rng = np.random.default_rng(7)
    rw, _, _ = synth.sample_reads(gw, n, 300, L, sub_rate=0.01, indel_rate=0.002, seed=41, mut_seed=42)
    reads = [unpack_symbols(host_u32(rw[i]), L).astype(np.uint8) for i in range(300)]
    for i in range(0, 300, 5):
        reads[i] = reads[i][:int(rng.integers(60, L))]
    reads += hand_reads(g, n, rng)
    return dict(O=O, g=g, gw=gw, idx=idx, fmi=fmi, reads=reads, n=n)


def read_set(reads, bits=2):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    return PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)


def params(band, typ, scheme, seed_len=20, seed_interval=10, max_seed_hits=20):
    return nb.SeedExtendParams(seed_len=seed_len, seed_interval=seed_interval, band_len=band, type=typ, both_strands=True,
                               max_seed_hits=max_seed_hits, scheme=scheme)


def hits_capacity(reads, p):
    return 2 * ((L - p.seed_len) // p.seed_interval + 1) * p.max_seed_hits * len(reads) + 1024     # every hit kept


def best_of(ws):
    torch.cuda.synchronize()
    return dict(best_score=ws.best_score.cpu().numpy().astype(np.int64), best_pos=host_u32(ws.best_pos).astype(np.int64),
                n_hits=ws.n_hits.cpu().numpy().astype(np.int64))


def assert_hits_equal(ws, want, what):
    torch.cuda.synchronize()
    kept, total, _ = [int(v) for v in ws.n_hits.cpu()]
    assert kept == total == want["n_hits"], what
    assert np.array_equal(ws.hit_read.cpu().numpy()[:kept].astype(np.int64), want["hit_string"]), what
    assert np.array_equal(host_u32(ws.hit_window)[:kept].astype(np.int64), want["hit_window"]), what
    assert np.array_equal(ws.hit_score.cpu().numpy()[:kept].astype(np.int64), want["hit_score"]), what
    assert np.array_equal(host_u32(ws.hit_sink)[:kept].astype(np.int64), want["hit_sink"]), what


def assert_best_equal(got, want, what):
    assert np.array_equal(got["best_score"], want["best_score"]), (what, np.flatnonzero(got["best_score"] != want["best_score"])[:8])
    assert np.array_equal(got["best_pos"], want["best_pos"]), (what, np.flatnonzero(got["best_pos"] != want["best_pos"])[:8])
    assert got["n_hits"][0] == got["n_hits"][1] == want["n_hits"], what


def overhang_rows(w, band):
    """indices of the hand-placed reads (both strands) that run more than band/2 symbols past the genome's end"""
    base = 300 + 4
    return [base + 2 * a + s for a, k in enumerate(OVERHANGS) if k > band // 2 for s in (0, 1)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# a. bands x types x schemes
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("band,typ", BAND_TYPES)
@pytest.mark.parametrize("scheme", SCHEMES, ids=repr)
def test_single_end_matrix(world, band, typ, scheme):
    w = world
    reads = w["reads"]
    p = params(band, typ, scheme)
    cap = hits_capacity(reads, p)
    rs = read_set(reads)
    want = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
    what = (band, typ, repr(scheme))
    # per-hit path: every hit
    ws = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap, keep_hits=True)
    assert_hits_equal(ws, want, what)
    assert_best_equal(best_of(ws), want, what + ("per hit",))
    # the reads past the genome's end by more than band/2: every job empty, the read unaligned
    for r in overhang_rows(w, band):
        assert want["best_score"][r] == INT_MIN and want["best_pos"][r] == NONE, (what, r)
    assert (want["hit_sink"][:, 0] == EMPTY_SINK).any(), what
    # per-read path: shortcut on, without its one-gap check, off
    eligible = typ == aln.LOCAL and band <= 32
    try:
        for sc in (1, 2, 0):
            _debug("nvb_debug_perfect_shortcut", sc)
            ws = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap)
            got = best_of(ws)
            assert_best_equal(got, want, what + ("shortcut %d" % sc,))
            if sc == 1 and eligible:
                dp = C.c_uint32(0)
                assert nb.lib().nvb_debug_dp_jobs(C.byref(dp)) == 0
                assert dp.value < got["n_hits"][2], what          # the shortcut claimed jobs
    finally:
        _debug("nvb_debug_perfect_shortcut", 1)


# ---------------------------------------------------------------------------------------------------------------------------------------
# b. seed geometry around a k = 10 table
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tables(world):
    """the world's index with a plain, a located and a context k = 10 table (the last with and without its per-row array)"""
    f = world["fmi"]
    out = {}
    for name, located, text in (("plain", False, None), ("located", True, None), ("context", True, world["gw"])):
        x = nb.FMIndexDevice(f.bwt_occ, f.ssa, f.L2, f.length, f.primary, sa_interval=1)
        x.build_ktab(10, located=located, text=text)
        out[name] = x
    assert out["context"].rows is not None
    torch.cuda.synchronize()
    return out


def geometry_reads(w):
    """2-bit: the first 200 world reads; 4-bit: 150 of them, ragged down to 4 symbols (shorter than any seed), with some N"""
    rng = np.random.default_rng(19)
    two = w["reads"][:200]
    four = []
    for i, r in enumerate(w["reads"][100:250]):
        r = r[:int(rng.integers(4, 19))].copy() if i % 6 == 0 else r.copy()
        r[rng.random(len(r)) < 0.004] = 4
        four.append(r)
    return two, four


@pytest.mark.parametrize("seed_len,seed_interval,max_seed_hits", [(8, 10, 8), (10, 10, 8), (11, 10, 8), (32, 10, 8), (20, 27, 8), (20, 10, 1)])
def test_seed_geometry(world, tables, seed_len, seed_interval, max_seed_hits):
    w = world
    sch = aln.SimpleGotohScheme(2, -2, -5, -3)
    p = params(31, aln.LOCAL, sch, seed_len=seed_len, seed_interval=seed_interval, max_seed_hits=max_seed_hits)
    for bits, reads in zip((2, 4), geometry_reads(w)):
        rs = read_set(reads, bits)
        cap = hits_capacity(reads, p)
        want = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
        what = (seed_len, seed_interval, max_seed_hits, bits)
        if bits == 4:
            short = [i for i, r in enumerate(reads) if len(r) < seed_len]
            assert short and all(want["best_score"][i] == INT_MIN for i in short)
        ws = nb.seed_extend(tables["plain"], w["gw"], rs, p, hit_capacity=cap, keep_hits=True)
        assert_hits_equal(ws, want, what)
        results = []
        for name in ("plain", "located", "context", "rows"):
            f = tables["context" if name == "rows" else name]
            rows = f.rows
            if name == "context":
                f.rows = None
            try:
                for split in (1, 0):
                    _debug("nvb_debug_seed_split", split)
                    got = best_of(nb.seed_extend(f, w["gw"], rs, p, hit_capacity=cap))
                    assert_best_equal(got, want, what + (name, split))
                    results.append(got)
            finally:
                _debug("nvb_debug_seed_split", 1)
                f.rows = rows
        for got in results[1:]:
            for k in got:
                assert np.array_equal(got[k], results[0][k]), what


# ---------------------------------------------------------------------------------------------------------------------------------------
# c. traceback across bands and types
# ---------------------------------------------------------------------------------------------------------------------------------------
def check_traceback(w, reads, p, best, ops, n_ops, begin, strand, want, what):
    """every read's alignment == the oracle's banded traceback of the read's best job (rebuilt from the oracle's winning hit); its ops
    replay to its score and end"""
    scheme6, _ = _scheme_args(p.scheme)
    bh = best_hits(want, len(reads))
    rows = np.flatnonzero(bh >= 0)
    for r in np.flatnonzero(bh < 0):
        assert n_ops[r] == 0 and tuple(begin[r]) == (NONE, NONE), (what, r)
    pats, t_off, t_len = [], [], []
    for r in rows:
        h = bh[r]
        s = int(want["hit_string"][h]) % 2
        pats.append(reads[r] if s == 0 else rc(reads[r]))
        t_off.append(int(want["hit_window"][h][0])); t_len.append(int(want["hit_window"][h][1] - want["hit_window"][h][0]))
        assert strand[r] == s, (what, r)
    lens = np.array([len(x) for x in pats], np.uint32)
    o = w["O"].banded_traceback(p.band_len, p.type, scheme6, np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens,
                                w["g"], np.array(t_off, np.uint32), np.array(t_len, np.uint32), max_ops=ops.shape[1])
    replayed = 0
    for a, r in enumerate(rows):
        assert n_ops[r] == o["n_ops"][a], (what, r)
        assert np.array_equal(ops[r, :n_ops[r]], o["ops"][a, :n_ops[r]]), (what, r)
        assert tuple(begin[r]) == (t_off[a] + int(o["source"][a][0]), int(o["source"][a][1])), (what, r)
        if int(best["best_pos"][r]) > w["n"]:
            continue                 # a GLOBAL band forced past the genome's end over pad symbols: the oracle's ops above are the check
        sc, e = replay(ops[r], n_ops[r], begin[r], pats[a], None, w["g"], p.scheme, typ=p.type, window=t_off[a])
        assert (sc, e) == (int(best["best_score"][r]), int(best["best_pos"][r])), (what, r)
        replayed += 1
    assert replayed > 0.8 * len(rows), what
    return len(rows)


@pytest.mark.parametrize("typ", [aln.GLOBAL, aln.LOCAL, aln.SEMI_GLOBAL])
@pytest.mark.parametrize("band", [3, 5, 7, 15, 31])
def test_traceback_matrix(world, band, typ):
    w = world
    reads = w["reads"]
    rs = read_set(reads)
    for scheme in (SCHEMES[0], SCHEMES[4]) if band == 15 else (SCHEMES[0],):
        p = params(band, typ, scheme)
        want = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
        ws = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=hits_capacity(reads, p), traceback=True)
        best = best_of(ws)
        what = (band, typ, repr(scheme))
        assert_best_equal(best, want, what)
        ops, n_ops = ws.best_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy()
        begin, strand = host_u32(ws.best_begin), ws.best_strand.cpu().numpy()
        checked = check_traceback(w, reads, p, best, ops, n_ops, begin, strand, want, what)
        assert checked > 0.8 * len(reads)
        for r in overhang_rows(w, band):
            assert n_ops[r] == 0 and tuple(begin[r]) == (NONE, NONE), (what, r)


def test_band_63_traceback_refused(world):
    """the banded traceback supports bands up to 31: band 63 is refused by the size query (its scoring runs, see the matrix above)"""
    w = world
    rs = read_set(w["reads"][:8])
    with pytest.raises(NvbError, match=r"\(-1\)"):
        nb.seed_extend(w["fmi"], w["gw"], rs, params(63, aln.LOCAL, SCHEMES[0]), hit_capacity=4096, traceback=True)
    ws = nb.seed_extend(w["fmi"], w["gw"], rs, params(63, aln.LOCAL, SCHEMES[0]), hit_capacity=4096)
    torch.cuda.synchronize()
    assert int(ws.n_hits[0]) > 0


# ---------------------------------------------------------------------------------------------------------------------------------------
# d. paired end-to-end and LOCAL at band 15
# ---------------------------------------------------------------------------------------------------------------------------------------
def pair_reads(w, n_pairs=200, Lp=100):
    """sampled FR pairs (some heavily mutated second mates, some second mates from another pair) plus pairs at the genome's start and
    end, the reverse mate running past the end by 5 .. 60 symbols"""
    g, n = w["g"], w["n"]
    rw, _, _ = synth.sample_pairs(w["gw"], n, n_pairs, Lp, frag_mean=300, frag_sd=40, sub_rate=0.02, hard_frac=0.3, hard_sub_rate=0.2,
                                  seed=51, mut_seed=52)
    reads = [unpack_symbols(host_u32(rw[i]), Lp).astype(np.uint8) for i in range(2 * n_pairs)]
    m1, m2 = reads[:n_pairs], reads[n_pairs:]
    m2[5:15] = [r.copy() for r in m2[105:115]]
    rng = np.random.default_rng(23)
    for k in (0, 5, 20, 40, 60):
        b = n - 300 + k
        frag = np.concatenate([g[b:], rng.integers(0, 4, k).astype(np.uint8)])
        m1.append(frag[:Lp].copy()); m2.append(rc(frag[-Lp:]))
    m1.append(g[:Lp].copy()); m2.append(rc(g[250:250 + Lp]))
    return m1 + m2, len(m1)


@pytest.mark.parametrize("mode", ["end_to_end", "local15"])
def test_paired_matrix(world, mode):
    w = world
    reads, n_pairs = pair_reads(w)
    Lp = max(len(r) for r in reads)
    if mode == "end_to_end":
        p = params(31, aln.SEMI_GLOBAL, aln.SimpleGotohScheme(0, -6, -5, -3), max_seed_hits=20)
        pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=-60)
        mq = nb.MapqParams.end_to_end(Lp)
    else:
        p = params(15, aln.LOCAL, aln.SimpleGotohScheme(2, -2, -5, -3), max_seed_hits=20)
        pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
        mq = nb.MapqParams.local(Lp)
    rs = read_set(reads)
    cap = hits_capacity(reads, p)
    ws = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap, mapq=mq, traceback=True)
    torch.cuda.synchronize()
    got = {k: getattr(ws, k).cpu().numpy().copy() for k in PAIR_KEYS + TB_KEYS + MAPQ_KEYS}
    # the same pair / MAPQ outputs from the calls without the traceback
    plain = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap)
    with_mapq = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap, mapq=mq)
    torch.cuda.synchronize()
    for k in PAIR_KEYS:
        assert np.array_equal(getattr(plain, k).cpu().numpy(), got[k]), (mode, k)
    for k in PAIR_KEYS + MAPQ_KEYS:
        assert np.array_equal(getattr(with_mapq, k).cpu().numpy(), got[k]), (mode, k)
    # pairs and MAPQ == the oracle composition
    want = pair_mapq_oracle(w["O"], w["idx"], w["g"], reads, p, pair, n_pairs, mq.min_score.cpu().numpy(), mq.match_bonus)
    assert tuple(int(v) for v in got["n_rescue"]) == tuple(want["n_rescue"]), mode
    for k in ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "second_pair_score", "second_mate_pos",
              "second_mate_strand", "mate_second_score", "mate_mapq"):
        g = got[k].astype(np.int64)
        if k in ("mate_pos", "second_mate_pos"):
            g = got[k].view(np.uint32).astype(np.int64)
        assert np.array_equal(g, want[k]), (mode, k, np.argwhere(g != want[k])[:6].tolist())
    pe = seed_extend_paired_oracle(w["O"], w["idx"], w["g"], reads, p, pair, n_pairs)
    for k in ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand"):
        assert np.array_equal(want[k], pe[k]), (mode, k)
    fl = want["pair_flags"]
    assert (fl == 1).sum() > 0.4 * n_pairs and ((fl == 2) | (fl == 4)).sum() > 10 and (fl == 0).sum() >= 5, mode
    # the pair whose reverse mate runs 60 symbols past the end: that mate has no alignment of its own (only empty jobs)
    se = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
    last = n_pairs - 2                                                      # (k = 60)
    assert se["best_score"][n_pairs + last] == INT_MIN and got["pair_flags"][last] != 1, mode
    # mates keeping their single-end best: nvb_seed_extend_traceback on the 2n reads
    single = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap, traceback=True)
    sbest = best_of(single)
    assert_best_equal(sbest, se, mode)
    s_ops, s_n, s_begin, s_strand = single.best_ops.cpu().numpy(), single.best_n_ops.cpu().numpy(), host_u32(single.best_begin), \
        single.best_strand.cpu().numpy()
    check_traceback(w, reads, p, sbest, s_ops, s_n, s_begin, s_strand, se, (mode, "single end"))
    flags, mops, mn, mbeg = got["pair_flags"], got["mate_ops"], got["mate_n_ops"], got["mate_begin"].view(np.uint32)
    rescued = []
    for q in range(n_pairs):
        for m in range(2):
            r = m * n_pairs + q
            if flags[q] in (2, 4) and m == (0 if flags[q] == 2 else 1):
                rescued.append((q, m))
                continue
            assert mn[m, q] == s_n[r] and tuple(mbeg[m, q]) == tuple(s_begin[r]), (mode, q, m)
            assert np.array_equal(mops[m, q, :mn[m, q]], s_ops[r, :s_n[r]]), (mode, q, m)
    assert rescued, mode
    # rescued mates: the oracle's full-matrix traceback of the winning opposite-mate job (pipeline_oracle's rule)
    scheme6, _ = _scheme_args(p.scheme)
    pats, t_off, t_len = [], [], []
    s_pos = sbest["best_pos"]
    for q, o in rescued:
        a = 1 - o
        ra, ro = a * n_pairs + q, o * n_pairs + q
        end = int(s_pos[ra]); beg = max(end - len(reads[ra]), 0)
        to, te = (beg, min(beg + pair.max_frag, w["n"])) if s_strand[ra] == 0 else (max(end - pair.max_frag, 0), end)
        pats.append(strand_string(reads[ro], np.zeros(len(reads[ro]), np.uint8), 1 - int(s_strand[ra]))[0])
        t_off.append(to); t_len.append(te - to)
    lens = np.array([len(x) for x in pats], np.uint32)
    o_ = w["O"].gotoh_full_traceback(p.type, scheme6, np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, w["g"],
                                     np.array(t_off, np.uint32), np.array(t_len, np.uint32), max_ops=ws.max_ops)
    for i, (q, o) in enumerate(rescued):
        assert int(o_["score"][i]) == got["mate_score"][o, q] and t_off[i] + int(o_["sink"][i][0]) == int(got["mate_pos"][o, q].view(np.uint32)), (mode, q, o)
        assert mn[o, q] == o_["n_ops"][i] and tuple(mbeg[o, q]) == (t_off[i] + int(o_["source"][i][0]), int(o_["source"][i][1])), (mode, q, o)
        assert np.array_equal(mops[o, q, :mn[o, q]], o_["ops"][i, :mn[o, q]]), (mode, q, o)
