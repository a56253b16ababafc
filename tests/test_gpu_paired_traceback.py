"""-m gpu: the alignment of both mates from paired-end seed + extend (nvb_seed_extend_paired_traceback) and the warp-per-alignment
full-matrix traceback behind its rescued mates (nvb_debug_full_traceback_warp).  Pair outputs equal nvb_seed_extend_paired[_mapq]; mates
that keep their own best equal nvb_seed_extend_traceback on the 2n reads; rescued mates equal the full-matrix traceback of the winning
opposite-mate job rebuilt by the rule of seed_extend_paired_oracle; every mate's ops replay to its score and end; and all of it is the
same on every path of the composition.  The argument validation needs no GPU."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200._lib import lib
from nvbio_b200.strings import PackedStringSet, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import _scheme_args

INT_MIN = -2**31
NONE = 0xFFFFFFFF


def _debug(name, v):
    getattr(lib(), name)(C.c_int(v))


@pytest.fixture(scope="module")
def world():
    """300 kbp genome, 500 pairs of 100 bp (30 % heavily mutated mates, 20 swapped second mates), indels in some mates (ragged lengths)"""
    require_gpu()
    O = orc.Oracle()
    n = 300_000
    gw = synth.random_genome_words(n, seed=78)
    gsym = unpack_symbols(host_u32(gw), n)
    idx = O.build_index(gsym)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    n_pairs, L = 500, 100
    rw, _, _ = synth.sample_pairs(gw, n, n_pairs, L, frag_mean=300, frag_sd=40, sub_rate=0.02, hard_frac=0.3, hard_sub_rate=0.2, seed=11, mut_seed=12)
    rw = rw.clone()
    rw[n_pairs + 5:n_pairs + 25] = rw[n_pairs + 105:n_pairs + 125].clone()
    reads = [unpack_symbols(host_u32(rw[i]), L).astype(np.uint8) for i in range(2 * n_pairs)]
    rng = np.random.default_rng(5)
    for i in rng.choice(2 * n_pairs, 200, replace=False):           # a 1-3 base deletion or insertion inside the read
        p, k = int(rng.integers(25, 75)), int(rng.integers(1, 4))
        r = reads[i]
        reads[i] = np.concatenate([r[:p], r[p + k:]]) if rng.random() < 0.5 else np.concatenate([r[:p], rng.integers(0, 4, k).astype(np.uint8), r[p:]])
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    return dict(O=O, idx=idx, gsym=gsym, gw=gw, fmi=fmi, n_pairs=n_pairs, reads=reads, quals=quals)


def read_set(w, bits=2):
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    return PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=bits, big_endian=True), offs


def make_params(w, qual=False, bits=2, dedup=True):
    if qual:
        _, offs = read_set(w, bits)
        q = torch.from_numpy(np.concatenate(w["quals"])).cuda()
        return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                                   dedup_jobs=dedup, scheme=aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3), read_quals=q)
    return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                               dedup_jobs=dedup, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


PAIR_KEYS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue")
TB_KEYS = ("mate_ops", "mate_n_ops", "mate_begin")
MAPQ_KEYS = ("second_pair_score", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")


def outputs(ws, keys):
    torch.cuda.synchronize()
    return {k: getattr(ws, k).cpu().numpy().copy() for k in keys}


def run(w, pair, bits=2, qual=False, dedup=True, mapq=None, traceback=True):
    rs, _ = read_set(w, bits)
    ws = nb.seed_extend_paired(w["fmi"], w["gw"], rs, make_params(w, qual, bits, dedup), pair, hit_capacity=64 * 2 * w["n_pairs"],
                               mapq=mapq, traceback=traceback)
    keys = PAIR_KEYS + (TB_KEYS if traceback else ()) + (MAPQ_KEYS if mapq is not None else ())
    return outputs(ws, keys), ws


def strand_string(r, q, strand):
    if strand == 0:
        return r, q
    return np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8), q[::-1]


def replay(ops, n_ops, begin, pat, pq, gsym, scheme, typ=aln.LOCAL, window=0):
    """score and genome end of an alignment (ops END->START) from its begin.  Both kinds of gap cost the pattern gap, as in the banded DP;
    a GLOBAL banded alignment that begins past its window's begin (genome coordinate `window`) also pays the text gap its first row
    starts with"""
    sch, tab = _scheme_args(scheme)
    match, mismatch, go, ge, tgo, tge = sch if len(sch) == 6 else sch + sch[2:]
    j, i = int(begin[0]), int(begin[1])
    s, prev = 0, -1
    if typ == aln.GLOBAL and j > window:
        s += tgo + (j - window - 1) * tge
    for op in ops[:n_ops][::-1]:
        if op == 0:
            eq = j < len(gsym) and pat[i] == gsym[j]                 # (a band running past the genome's end meets pad symbols)
            s += (int(tab[pq[i], 0 if eq else 1]) if tab is not None else (match if eq else mismatch)); i += 1; j += 1
        elif op == 1:
            s += ge if prev == 1 else go; i += 1
        else:
            s += ge if prev == 2 else go; j += 1
        prev = op
    return s, j


@pytest.mark.gpu
@pytest.mark.parametrize("qual", [False, True])
def test_paired_traceback_vs_single_end_and_rescue_jobs(world, qual):
    w = world
    n_pairs, reads, quals = w["n_pairs"], w["reads"], w["quals"]
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    got, ws = run(w, pair, qual=qual)
    plain, _ = run(w, pair, qual=qual, traceback=False)
    for k in PAIR_KEYS:
        assert np.array_equal(got[k], plain[k]), k
    mp = nb.MapqParams.local(max(len(r) for r in reads))
    with_mapq, _ = run(w, pair, qual=qual, mapq=mp)
    ref_mapq, _ = run(w, pair, qual=qual, mapq=mp, traceback=False)
    for k in PAIR_KEYS + MAPQ_KEYS:
        assert np.array_equal(with_mapq[k], ref_mapq[k]), k
    for k in TB_KEYS:
        assert np.array_equal(with_mapq[k], got[k]), k

    # single end on the 2n reads
    rs, offs = read_set(w)
    params = make_params(w, qual)
    se = nb.seed_extend(w["fmi"], w["gw"], rs, params, hit_capacity=64 * 2 * n_pairs, traceback=True)
    torch.cuda.synchronize()
    se_ops, se_n, se_begin = se.best_ops.cpu().numpy(), se.best_n_ops.cpu().numpy(), host_u32(se.best_begin)
    se_pos, se_strand = host_u32(se.best_pos), se.best_strand.cpu().numpy()
    flags, mops, mn, mbeg = got["pair_flags"], got["mate_ops"], got["mate_n_ops"], got["mate_begin"].view(np.uint32)
    max_ops = ws.max_ops
    rescued = []
    for p in range(n_pairs):
        for m in range(2):
            r = m * n_pairs + p
            if flags[p] in (2, 4) and m == (0 if flags[p] == 2 else 1):
                rescued.append((p, m))
                continue
            assert mn[m, p] == se_n[r] and np.array_equal(mbeg[m, p], se_begin[r]), (p, m)
            assert np.array_equal(mops[m, p, :min(mn[m, p], max_ops)], se_ops[r, :min(se_n[r], max_ops)]), (p, m)
            if got["mate_pos"][m, p] == -1:
                assert mn[m, p] == 0 and tuple(mbeg[m, p]) == (NONE, NONE)
    assert len(rescued) > 0.1 * n_pairs

    # rescued mates: the winning opposite-mate job rebuilt (pipeline_oracle's rule), traced by nvb_gotoh_traceback on its whole window
    glen = w["idx"].n
    pats, pq, t_off, t_len = [], [], [], []
    for p, o in rescued:
        a = 1 - o
        ra, ro = a * n_pairs + p, o * n_pairs + p
        end = int(se_pos[ra]); beg = max(end - len(reads[ra]), 0)
        if se_strand[ra] == 0:
            to, te = beg, min(beg + pair.max_frag, glen)
        else:
            to, te = max(end - pair.max_frag, 0), end
        pt, qt = strand_string(reads[ro], quals[ro], 1 - int(se_strand[ra]))
        pats.append(pt); pq.append(qt); t_off.append(to); t_len.append(te - to)
    lens = np.array([len(x) for x in pats], np.uint32)
    P = PackedStringSet.from_symbols(np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, bits=2)
    T = PackedStringSet.from_symbols(w["gsym"], np.array(t_off, np.uint32), np.array(t_len, np.uint32), bits=2)
    qt = torch.from_numpy(np.concatenate(pq)).cuda() if qual else None
    want = aln.batch_alignment_traceback(aln.make_gotoh_aligner(aln.LOCAL, params.scheme), P, T, max_ops=max_ops, quals=qt)
    torch.cuda.synchronize()
    ws_ops, ws_n, ws_src, ws_sink = want["ops"].cpu().numpy(), host_u32(want["n_ops"]), host_u32(want["source"]), host_u32(want["sink"])
    ws_score = want["score"].cpu().numpy()
    for i, (p, o) in enumerate(rescued):
        assert ws_score[i] == got["mate_score"][o, p] and t_off[i] + ws_sink[i][0] == got["mate_pos"][o, p].astype(np.uint32)
        assert mn[o, p] == ws_n[i] and tuple(mbeg[o, p]) == (t_off[i] + ws_src[i][0], ws_src[i][1]), (p, o)
        assert np.array_equal(mops[o, p, :min(ws_n[i], max_ops)], ws_ops[i, :min(ws_n[i], max_ops)]), (p, o)

    # every aligned mate's ops replay to its score and end; both kinds of gap occur
    seen = set()
    for p in range(n_pairs):
        for m in range(2):
            if got["mate_pos"][m, p] == -1:
                continue
            r = m * n_pairs + p
            assert mn[m, p] <= max_ops
            pat, q = strand_string(reads[r], quals[r], int(got["mate_strand"][m, p]))
            s, e = replay(mops[m, p], mn[m, p], mbeg[m, p], pat, q, w["gsym"], params.scheme)
            assert (s, e) == (int(got["mate_score"][m, p]), int(got["mate_pos"][m, p])), (p, m)
            seen |= set(int(v) for v in mops[m, p, :mn[m, p]])
    assert seen == {0, 1, 2}


@pytest.mark.gpu
def test_paired_traceback_same_on_every_path(world):
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    base, _ = run(w, pair)
    variants = []
    try:
        _debug("nvb_debug_pipeline_path", 1); variants.append(("per-hit", run(w, pair)[0]))
        _debug("nvb_debug_pipeline_path", 0)
        variants.append(("dedup off", run(w, pair, dedup=False)[0]))
        for sc in (0, 2):
            _debug("nvb_debug_perfect_shortcut", sc); variants.append(("shortcut %d" % sc, run(w, pair)[0]))
        _debug("nvb_debug_perfect_shortcut", 1)
        _debug("nvb_debug_seed_split", 0); variants.append(("seed split 0", run(w, pair)[0]))
        _debug("nvb_debug_seed_split", 1)
        variants.append(("4-bit", run(w, pair, bits=4)[0]))
    finally:
        _debug("nvb_debug_pipeline_path", 0); _debug("nvb_debug_perfect_shortcut", 1); _debug("nvb_debug_seed_split", 1)
    for name, v in variants:
        for k in PAIR_KEYS + TB_KEYS:
            assert np.array_equal(v[k], base[k]), (name, k)
    # a capacity-limited rescue: pair outputs as without the traceback
    small = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50, rescue_capacity=37)
    got, _ = run(w, small)
    plain, _ = run(w, small, traceback=False)
    for k in PAIR_KEYS:
        assert np.array_equal(got[k], plain[k]), k


@pytest.mark.gpu
def test_single_end_traceback_per_read_equals_per_hit(world):
    w = world
    rs, _ = read_set(w)
    outs = []
    try:
        for path in (0, 1):
            for sc in (1, 0):
                _debug("nvb_debug_pipeline_path", path); _debug("nvb_debug_perfect_shortcut", sc)
                se = nb.seed_extend(w["fmi"], w["gw"], rs, make_params(w), hit_capacity=64 * len(w["reads"]), traceback=True)
                outs.append([t.cpu().numpy().copy() for t in (se.best_score, se.best_pos, se.best_ops, se.best_n_ops, se.best_begin, se.best_strand)])
    finally:
        _debug("nvb_debug_pipeline_path", 0); _debug("nvb_debug_perfect_shortcut", 1)
    for o in outs[1:]:
        for a, b in zip(o, outs[0]):
            assert np.array_equal(a, b)


def _random_batch(rng, n, max_m, max_n, pbits):
    p_len = rng.integers(1, max_m + 1, n).astype(np.uint32)
    t_len = rng.integers(1, max_n + 1, n).astype(np.uint32)
    txt = rng.integers(0, 4, int(t_len.sum())).astype(np.uint8)
    t_off = np.concatenate([[0], np.cumsum(t_len)[:-1]]).astype(np.uint32)
    pats = []
    for a in range(n):                     # half the patterns come from their text (mutated, with indels), half are random
        if rng.random() < 0.5 and t_len[a] >= p_len[a]:
            s = int(rng.integers(0, t_len[a] - p_len[a] + 1))
            q = txt[t_off[a] + s:t_off[a] + s + p_len[a]].copy()
            mut = rng.random(len(q)) < 0.08
            q[mut] = rng.integers(0, 4, int(mut.sum()))
            if len(q) > 10 and rng.random() < 0.5:
                k = int(rng.integers(1, len(q) - 5)); q = np.concatenate([q[:k], q[k + 2:], rng.integers(0, 4, 2).astype(np.uint8)])
        else:
            q = rng.integers(0, 4, int(p_len[a])).astype(np.uint8)
        if rng.random() < 0.3 and len(q) >= 2:
            q = np.tile(q[:int(rng.choice([1, 2, 7]))], len(q))[:len(q)]           # tandem repeats
        pats.append(q.astype(np.uint8))
    pat = np.concatenate(pats)
    if pbits == 4:
        pat[rng.integers(0, len(pat), max(1, len(pat) // 50))] = 4                     # N's
    p_off = np.concatenate([[0], np.cumsum(p_len)[:-1]]).astype(np.uint32)
    return pat, p_off, p_len, txt, t_off, t_len


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [aln.GLOBAL, aln.LOCAL, aln.SEMI_GLOBAL])
def test_warp_traceback_equals_default_path(typ):
    """nvb_gotoh_traceback through the warp kernel (nvb_debug_full_traceback_warp(1)) == the default kernel (and the reference where it is
    built), every output, on random batches: M 1..512 (every W at its boundaries), N up to 1000, N symbols, quality tables, and a batch
    larger than the slot pool"""
    require_gpu()
    rng = np.random.default_rng(40 + typ)
    schemes = [aln.SimpleGotohScheme(2, -2, -5, -3), aln.SimpleGotohScheme(1, -3, -4, -1), aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3)]
    R = orc.Ref() if orc.Ref.available() else None
    cases = [(m, 200) for m in (1, 2, 31, 32, 33, 64, 65, 96, 97, 128, 129, 255, 256, 257, 288, 289, 320, 321, 352, 353, 384, 385,
                                 416, 417, 448, 449, 480, 481, 511, 512)]
    cases += [(150, 1000), (100, 500), (20, 40)]
    for (max_m, max_n) in cases:
        n = 30000 if max_m == 20 else 64
        for si, sch in enumerate(schemes):
            if max_m == 20 and si != 2:
                continue
            pbits = 4 if si == 1 else 2
            pat, p_off, p_len, txt, t_off, t_len = _random_batch(rng, n, max_m, max_n, pbits)
            P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits)
            T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2)
            q = torch.from_numpy(rng.integers(0, 45, len(pat)).astype(np.uint8)).cuda() if si == 2 else None
            al = aln.make_gotoh_aligner(typ, sch)
            outs = []
            try:
                for mode in (0, 1):
                    _debug("nvb_debug_full_traceback_warp", mode)
                    o = aln.batch_alignment_traceback(al, P, T, max_ops=max_m + max_n + 1, quals=q)
                    torch.cuda.synchronize()
                    outs.append({k: v.cpu().numpy() for k, v in o.items()})
            finally:
                _debug("nvb_debug_full_traceback_warp", 0)
            for k in ("score", "sink", "source", "n_ops", "ops"):
                assert np.array_equal(outs[1][k], outs[0][k]), (max_m, max_n, si, k)
            if R is not None and si == 0 and max_m <= 256 and max_n <= 512:
                want = R.gotoh_full_traceback(typ, (2, -2, -5, -3), pat, p_off, p_len, txt, t_off, t_len, max_ops=max_m + max_n + 1)
                for k in ("score", "n_ops"):
                    assert np.array_equal(outs[1][k].astype(np.int64), want[k].astype(np.int64)), (max_m, k)


def test_argument_validation_without_gpu():
    """nvb_seed_extend_paired_traceback: NVB_E_INVALID (-1) for a missing or incomplete mate_alignment, mapq without mapq_out (or the
    reverse) and every failed check of the paired calls; NVB_E_UNSUPPORTED (-4) for reads longer than 512 -- all before any CUDA call"""
    from nvbio_b200._lib import (StringSetStruct, GotohSchemeStruct, PairParamsStruct, PairOutStruct, SeedExtendParamsStruct, FmIndexStruct,
                                 BestAlignmentOutStruct, MapqParamsStruct, PairMapqOutStruct)
    L = lib()
    f = L.nvb_seed_extend_paired_traceback
    tb = C.c_size_t(0)
    ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    pp = PairParamsStruct(); pp.min_frag, pp.max_frag, pp.min_mate_score, pp.rescue_capacity = 0, 500, 50, 100
    po = PairOutStruct()
    for k in ("d_pair_score", "d_pair_flags", "d_mate_score", "d_mate_pos", "d_mate_strand"):
        setattr(po, k, 16)
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    ba = BestAlignmentOutStruct(); ba.d_ops = 16; ba.max_ops = 300; ba.d_n_ops = 16; ba.d_begin = 16
    mp = MapqParamsStruct(); mp.d_min_score = 16; mp.max_read_len = 150; mp.match_bonus = 2
    mo = PairMapqOutStruct(); mo.d_second_pair_score = 16; mo.d_mate_mapq = 16

    def call(ba_=ba, mp_=mp, mo_=mo, ss_=ss, sp_=sp, po_=po, pp_=pp, fm_=fm, genome=16, tb_=tb, n_pairs=8):
        r = lambda x: C.byref(x) if x is not None else None      # noqa: E731
        return f(r(fm_), C.c_void_p(genome), r(ss_), C.c_uint32(n_pairs), r(sp_), C.c_uint32(100), r(pp_), r(po_), r(ba_), r(mp_), r(mo_),
                 None, None, r(tb_), None)
    assert call(ba_=None) == -1
    for k in ("d_ops", "d_n_ops", "d_begin"):
        b = BestAlignmentOutStruct(); b.d_ops = 16; b.max_ops = 300; b.d_n_ops = 16; b.d_begin = 16
        setattr(b, k, None)
        assert call(ba_=b) == -1, k
    b = BestAlignmentOutStruct(); b.d_ops = 16; b.max_ops = 0; b.d_n_ops = 16; b.d_begin = 16
    assert call(ba_=b) == -1
    assert call(mo_=None) == -1 and call(mp_=None) == -1
    short = MapqParamsStruct(); short.d_min_score = 16; short.max_read_len = 100; short.match_bonus = 2
    assert call(mp_=short) == -1
    bad_out = PairOutStruct()
    assert call(po_=bad_out) == -1
    sp1 = SeedExtendParamsStruct(); sp1.seed_len, sp1.seed_interval, sp1.band_len, sp1.type, sp1.both_strands, sp1.max_seed_hits = 20, 10, 31, 1, 0, 100
    sp1.scheme = sch
    assert call(sp_=sp1) == -1
    long_ = StringSetStruct(); long_.d_words = 16; long_.bits = 2; long_.big_endian = 1; long_.stride = 528; long_.length = 513
    assert call(ss_=long_, mp_=None, mo_=None) == -4
    assert call(ss_=None) == -1 and call(tb_=None) == -1 and call(pp_=None) == -1 and call(po_=None) == -1 and call(n_pairs=0x40000000) == -1
    # which code wins when several checks fail: the call's arguments, mate_alignment and the MAPQ inputs / outputs (-1), then reads over
    # 512 bp (-4), then the pair outputs and parameters and the index, reads and seed parameters (-1 or -4)
    big = MapqParamsStruct(); big.d_min_score = 16; big.max_read_len = 513; big.match_bonus = 2
    for k in ("d_ops", "d_n_ops", "d_begin", "max_ops"):
        b = BestAlignmentOutStruct(); b.d_ops = 16; b.max_ops = 300; b.d_n_ops = 16; b.d_begin = 16
        setattr(b, k, None if k != "max_ops" else 0)
        assert call(ss_=long_, ba_=b, mp_=big) == -1, k
    assert call(ss_=long_, ba_=None) == -1 and call(ss_=long_, tb_=None) == -1 and call(ss_=long_, pp_=None) == -1
    assert call(ss_=long_, po_=None) == -1 and call(ss_=long_, n_pairs=0x40000000) == -1
    assert call(ss_=long_, mp_=big, mo_=None) == -1 and call(ss_=long_, mp_=None) == -1
    assert call(ss_=long_) == -1                                          # the min-score table (150) does not cover 513
    assert call(ss_=long_, mp_=big) == -4
    no_min = MapqParamsStruct(); no_min.max_read_len = 513; no_min.match_bonus = 2
    assert call(ss_=long_, mp_=no_min) == -1
    no_mapq = PairMapqOutStruct(); no_mapq.d_second_pair_score = 16
    assert call(ss_=long_, mp_=big, mo_=no_mapq) == -1
    assert call(ss_=long_, mp_=big, po_=bad_out) == -4 and call(ss_=long_, mp_=big, sp_=sp1) == -4
    far = PairParamsStruct(); far.min_frag, far.max_frag, far.min_mate_score, far.rescue_capacity = 600, 500, 50, 100
    assert call(ss_=long_, mp_=big, pp_=far) == -4 and call(pp_=far) == -1
    bad_fm = FmIndexStruct(); bad_fm.d_bwt_occ = 32; bad_fm.d_ssa = 32; bad_fm.length = 1000; bad_fm.primary = 5; bad_fm.sa_interval = 12
    assert call(ss_=long_, mp_=big, fm_=bad_fm) == -4 and call(fm_=bad_fm) == -1
    assert call(ss_=long_, mp_=big, genome=None) == -4 and call(genome=None) == -1
    assert call(ss_=long_, mp_=big, sp_=None) == -4 and call(sp_=None) == -1
    long8 = StringSetStruct(); long8.d_words = 16; long8.bits = 8; long8.big_endian = 1; long8.stride = 528; long8.length = 513
    assert call(ss_=long8, mp_=None, mo_=None) == -4 and call(ss_=long8, mp_=None, mo_=None, po_=bad_out) == -4
    # 8-bit reads (-4) lose to every failed paired, best-alignment and MAPQ check
    s8 = StringSetStruct(); s8.d_words = 16; s8.bits = 8; s8.big_endian = 1; s8.stride = 152; s8.length = 150
    assert call(ss_=s8) == -4
    no_ops = BestAlignmentOutStruct(); no_ops.d_ops = 16; no_ops.max_ops = 0; no_ops.d_n_ops = 16; no_ops.d_begin = 16
    assert call(ss_=s8, po_=bad_out) == -1 and call(ss_=s8, sp_=sp1) == -1 and call(ss_=s8, pp_=far) == -1 and call(ss_=s8, ba_=no_ops) == -1
    assert call(ss_=s8, mp_=short) == -1 and call(ss_=s8, mo_=None) == -1 and call(ss_=s8, mo_=no_mapq) == -1
