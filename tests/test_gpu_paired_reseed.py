"""-m gpu: reseeding rounds before pairing (nvb_seed_extend_paired_reseed) on a genome with a planted 16-copy family
(tests/paired_reseed_oracle.py's world): bit-identical to nvb_seed_extend_paired[_mapq|_traceback] at max_reseed 0, the composed oracle
at 1 to 3 rounds on every path and configuration, the effect on substitution and in-family pairs, the mate tracebacks, the BAM chain and
the argument checks."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200._lib import lib, ReseedOutStruct, PairOutStruct
from nvbio_b200.pipeline import MapqParams, ReseedParams
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.paired_reseed_oracle import seed_extend_paired_reseed_oracle, planted_pairs, CLASSES, RL, L, I, rc

pytestmark = pytest.mark.gpu

INT_MIN = -2**31
NONE = 0xFFFFFFFF
REP = 8
PAIR_KEYS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue")
MAPQ_KEYS = ("second_pair_score", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")
TB_KEYS = ("mate_ops", "mate_n_ops", "mate_begin")
U32_KEYS = ("mate_pos", "second_mate_pos")


@pytest.fixture(scope="module")
def world():
    require_gpu()
    O = orc.Oracle()
    g, reads, cls, truth = planted_pairs()
    G = len(g)
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    fmi_loc = nb.FMIndexDevice.from_text(gw, G, sa_interval=1)[0]
    fmi_loc.build_ktab(8, located=True, text=gw)
    return dict(O=O, g=g, G=G, gw=gw, idx=idx, fmi=fmi, fmi_loc=fmi_loc, reads=reads, cls=cls, truth=truth, n_pairs=len(cls))


def packed(reads, bits=2):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = (np.cumsum(lens) - lens).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)
    rs.length = RL
    return rs


def params_for(typ, qual=None, hits=4, dedup=True):
    if qual is not None:
        sch = aln.QualityGotohScheme(2 if typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3)
    else:
        sch = aln.SimpleGotohScheme(2, -2, -5, -3) if typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
    return nb.SeedExtendParams(seed_len=L, seed_interval=I, band_len=15, type=typ, both_strands=True, max_seed_hits=hits, scheme=sch,
                               read_quals=qual, dedup_jobs=dedup)


def pair_for(typ, rescue_capacity=None):
    return nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60 if typ == aln.LOCAL else -60, rescue_capacity=rescue_capacity)


def tables(typ, max_reseed):
    mq = MapqParams.local(RL) if typ == aln.LOCAL else MapqParams.end_to_end(RL)
    return mq, ReseedParams(mq.min_score, max_reseed, REP)


def outs(ws, keys):
    torch.cuda.synchronize()
    o = {}
    for k in keys:
        a = getattr(ws, k).cpu().numpy()
        o[k] = (a.view(np.uint32) if k in U32_KEYS else a).astype(np.int64)
    return o


def _debug(name, v):
    getattr(lib(), name)(C.c_int(v))


def test_max_reseed_zero_is_the_paired_calls(world):
    """max_reseed 0: every output bit-identical to nvb_seed_extend_paired / _paired_mapq / _paired_traceback, on the per-read and the
    per-hit path, on both index formats"""
    w = world
    rs = packed(w["reads"])
    cap = 64 * rs.count
    for typ in (aln.LOCAL, aln.SEMI_GLOBAL):
        p, pair = params_for(typ), pair_for(typ)
        mq, rp = tables(typ, 0)
        for path in (0, 1):
            _debug("nvb_debug_pipeline_path", path)
            try:
                for fmi in (w["fmi"], w["fmi_loc"]):
                    for tb, m in ((False, None), (False, mq), (True, None), (True, mq)):
                        a = nb.seed_extend_paired(fmi, w["gw"], rs, p, pair, hit_capacity=cap, mapq=m, traceback=tb)
                        b = nb.seed_extend_paired_reseed(fmi, w["gw"], rs, p, pair, rp, mapq=m, traceback=tb, hit_capacity=cap)
                        torch.cuda.synchronize()
                        for k in PAIR_KEYS + MAPQ_KEYS + TB_KEYS + ("n_hits",):
                            x, y = getattr(a, k), getattr(b, k)
                            assert (x is None) == (y is None), k
                            if x is not None:
                                assert torch.equal(x, y), (typ, path, tb, m is not None, k)
                        assert (b.rounds == 1).all() and b.active.tolist() == [rs.count]
            finally:
                _debug("nvb_debug_pipeline_path", 0)


CONFIGS = [(2, aln.LOCAL, False), (4, aln.LOCAL, False), (2, aln.SEMI_GLOBAL, False), (2, aln.LOCAL, True)]


def config_inputs(w, bits, qual):
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        rng = np.random.default_rng(5)
        for r in reads[3::7]:
            r[rng.integers(0, len(r), 1)] = 4                     # N
    quals = qt = None
    if qual:
        rng = np.random.default_rng(9)
        quals = [rng.integers(0, 45, len(r)).astype(np.uint8) for r in reads]
        qt = torch.from_numpy(np.concatenate(quals)).cuda()
    return reads, quals, qt


def check(ws, want, keys, what):
    got = outs(ws, keys)
    for k in keys:
        w_ = np.asarray(want[k], np.int64)
        bad = np.argwhere(got[k] != w_)
        assert len(bad) == 0, (what, k, [(tuple(int(v) for v in i), int(got[k][tuple(i)]), int(w_[tuple(i)])) for i in bad[:5]])
    got = outs(ws, ("rounds", "active"))
    assert np.array_equal(got["rounds"], want["rounds"]) and np.array_equal(got["active"], want["active"]), what
    assert host_u32(ws.n_hits)[:2].tolist() == list(want["n_hits"]), what


@pytest.mark.parametrize("max_reseed", [1, 2, 3])
@pytest.mark.parametrize("bits,typ,qual", CONFIGS)
def test_vs_oracle(world, max_reseed, bits, typ, qual):
    w = world
    reads, quals, qt = config_inputs(w, bits, qual)
    rs = packed(reads, bits)
    p, pair = params_for(typ, qt), pair_for(typ)
    mq, rp = tables(typ, max_reseed)
    cap = 64 * rs.count
    want = seed_extend_paired_reseed_oracle(w["O"], w["idx"], w["g"], reads, p, pair, w["n_pairs"], max_reseed, REP, cap,
                                            min_score=mq.min_score.cpu().numpy(), match_bonus=mq.match_bonus, quals=quals)
    assert want["active"][0] == len(reads) and want["active"][1] > 0
    # per-read path (default), both index formats, with and without MAPQ
    for fmi in (w["fmi"], w["fmi_loc"]):
        check(nb.seed_extend_paired_reseed(fmi, w["gw"], rs, p, pair, rp, hit_capacity=cap), want, PAIR_KEYS, "per-read")
        check(nb.seed_extend_paired_reseed(fmi, w["gw"], rs, p, pair, rp, mapq=mq, hit_capacity=cap), want, PAIR_KEYS + MAPQ_KEYS,
              "per-read mapq")
    # the exact shortcut at 0 / 2 (1 above), the seed split off
    for name, val, dflt in (("nvb_debug_perfect_shortcut", 0, 1), ("nvb_debug_perfect_shortcut", 2, 1), ("nvb_debug_seed_split", 0, 1)):
        _debug(name, val)
        try:
            check(nb.seed_extend_paired_reseed(w["fmi_loc"], w["gw"], rs, p, pair, rp, mapq=mq, hit_capacity=cap), want,
                  PAIR_KEYS + MAPQ_KEYS, (name, val))
        finally:
            _debug(name, dflt)
    # per-hit path, with and without de-duplication
    _debug("nvb_debug_pipeline_path", 1)
    try:
        for dedup in (True, False):
            p.dedup_jobs = dedup
            check(nb.seed_extend_paired_reseed(w["fmi"], w["gw"], rs, p, pair, rp, mapq=mq, hit_capacity=cap), want,
                  PAIR_KEYS + MAPQ_KEYS, ("per-hit", dedup))
    finally:
        _debug("nvb_debug_pipeline_path", 0)
        p.dedup_jobs = True


def test_capacities(world):
    """a hit capacity that overflows in round 1, and a rescue capacity that cuts the rescue"""
    w = world
    rs = packed(w["reads"])
    p = params_for(aln.LOCAL)
    mq, rp = tables(aln.LOCAL, 2)
    ws0 = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair_for(aln.LOCAL), hit_capacity=64 * rs.count)
    torch.cuda.synchronize()
    for cap, pair in ((int(ws0.n_hits[0]) + 40, pair_for(aln.LOCAL)), (64 * rs.count, pair_for(aln.LOCAL, rescue_capacity=1))):
        want = seed_extend_paired_reseed_oracle(w["O"], w["idx"], w["g"], w["reads"], p, pair, w["n_pairs"], 2, REP, cap,
                                                min_score=mq.min_score.cpu().numpy(), match_bonus=mq.match_bonus)
        if pair.rescue_capacity is None:
            assert want["n_hits"][0] == cap and want["n_hits"][1] > cap
        else:
            assert want["n_rescue"][0] == 1 and want["n_rescue"][1] > 1
        for path in (0, 1):
            _debug("nvb_debug_pipeline_path", path)
            try:
                check(nb.seed_extend_paired_reseed(w["fmi"], w["gw"], rs, p, pair, rp, mapq=mq, hit_capacity=cap), want,
                      PAIR_KEYS + MAPQ_KEYS, (cap, pair.rescue_capacity, path))
            finally:
                _debug("nvb_debug_pipeline_path", 0)


def replay(ops, n_ops, begin, pat, g):
    """score and genome end of a LOCAL 2 / -2 / 5 / 3 alignment (ops END->START) from its begin"""
    t, q, score, prev = int(begin[0]), int(begin[1]), 0, -1
    for o in ops[:n_ops][::-1]:
        if o == 0:
            score += 2 if pat[q] == g[t] else -2; q += 1; t += 1
        elif o == 1:
            score -= 5 if prev != 1 else 3; q += 1
        else:
            score -= 5 if prev != 2 else 3; t += 1
        prev = o
    return score, t


def test_effect_traceback_and_bam(world):
    w = world
    n, reads, cls, truth = w["n_pairs"], w["reads"], w["cls"], w["truth"]
    rs = packed(reads)
    p, pair = params_for(aln.LOCAL), pair_for(aln.LOCAL)
    mq, rp0 = tables(aln.LOCAL, 0)
    _, rp2 = tables(aln.LOCAL, 2)
    ws0 = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], rs, p, pair, rp0, mapq=mq, traceback=True)
    ws2 = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], rs, p, pair, rp2, mapq=mq, traceback=True)
    keys = PAIR_KEYS + MAPQ_KEYS + TB_KEYS + ("rounds",)
    o0, o2 = outs(ws0, keys), outs(ws2, keys)
    lens = np.array([len(r) for r in reads]).reshape(2, n)
    near = lambda o, q: np.abs(o["mate_pos"][:, q] - lens[:, q] - truth[q].T) <= 4          # noqa: E731
    at = lambda o, q: o["mate_pos"][:, q] == truth[q].T + lens[:, q]                        # noqa: E731

    # both mates under substitutions: no anchor without reseeding, concordant at the locus with it
    q = np.flatnonzero(cls == CLASSES.index("sub2"))
    assert (o0["pair_flags"][q] == nb.pipeline.PAIR_UNPAIRED).all() and (o0["mate_score"][:, q] == INT_MIN).all()
    assert (o2["pair_flags"][q] == nb.pipeline.PAIR_CONCORDANT).all() and near(o2, q).all()
    # one such mate: rescued without reseeding, concordant with it
    q = np.flatnonzero(cls == CLASSES.index("sub1"))
    assert (o0["pair_flags"][q] == nb.pipeline.PAIR_RESCUED_MATE1).all()
    assert (o2["pair_flags"][q] == nb.pipeline.PAIR_CONCORDANT).all() and near(o2, q).all()
    # in-family pairs: at their own copy with reseeding, not all of them without
    q = np.flatnonzero(cls == CLASSES.index("family"))
    assert (o2["pair_flags"][q] == nb.pipeline.PAIR_CONCORDANT).all() and at(o2, q).all()
    assert not ((o0["pair_flags"][q] == nb.pipeline.PAIR_CONCORDANT) & at(o0, q).all(axis=0)).all()

    # every traced mate replays to its score and end
    g = w["g"]
    for m in range(2):
        for i in range(n):
            if o2["mate_pos"][m, i] == NONE:
                assert o2["mate_n_ops"][m, i] == 0
                continue
            r = reads[m * n + i]
            pat = r if o2["mate_strand"][m, i] == 0 else rc(r)
            assert replay(o2["mate_ops"][m, i], o2["mate_n_ops"][m, i], o2["mate_begin"][m, i], pat, g) == \
                (o2["mate_score"][m, i], o2["mate_pos"][m, i]), (m, i)

    # rescued mates: the winning opposite-mate job rebuilt from its anchor (pipeline_oracle's rule), traced by nvb_gotoh_traceback
    resc = [(i, 0 if o2["pair_flags"][i] == 2 else 1) for i in np.flatnonzero(np.isin(o2["pair_flags"], (2, 4)))]
    assert resc
    pats, t_off, t_len = [], [], []
    for i, o in resc:
        a = 1 - o
        end = int(o2["mate_pos"][a, i]); beg = max(end - len(reads[a * n + i]), 0)
        to, te = (beg, min(beg + pair.max_frag, w["G"])) if o2["mate_strand"][a, i] == 0 else (max(end - pair.max_frag, 0), end)
        r = reads[o * n + i]
        pats.append(rc(r) if o2["mate_strand"][a, i] == 0 else r); t_off.append(to); t_len.append(te - to)
    plen = np.array([len(x) for x in pats], np.uint32)
    P = PackedStringSet.from_symbols(np.concatenate(pats), np.concatenate([[0], np.cumsum(plen)[:-1]]).astype(np.uint32), plen, bits=2)
    T = PackedStringSet.from_symbols(g, np.array(t_off, np.uint32), np.array(t_len, np.uint32), bits=2)
    tb = aln.batch_alignment_traceback(aln.make_gotoh_aligner(aln.LOCAL, p.scheme), P, T, max_ops=ws2.max_ops)
    torch.cuda.synchronize()
    t_ops, t_n, t_src, t_sink = tb["ops"].cpu().numpy(), host_u32(tb["n_ops"]), host_u32(tb["source"]), host_u32(tb["sink"])
    t_score = tb["score"].cpu().numpy()
    for j, (i, o) in enumerate(resc):
        assert t_score[j] == o2["mate_score"][o, i] and t_off[j] + t_sink[j][0] == o2["mate_pos"][o, i], (i, o)
        assert o2["mate_n_ops"][o, i] == t_n[j] and tuple(o2["mate_begin"][o, i]) == (t_off[j] + t_src[j][0], t_src[j][1]), (i, o)
        assert np.array_equal(o2["mate_ops"][o, i, :t_n[j]], t_ops[j, :t_n[j]]), (i, o)

    # pairs whose mates were both seeded once: the same records with and without reseeding
    contigs = nb.ContigTable(["chr1"], [w["G"]])
    names = nb.numbered_names(n)

    def records(ws):
        f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=w["G"])
        recs = nb.bam_records(ws, f, rs, contigs, names)
        off = recs.offsets.cpu().numpy()
        data = recs.to_bytes()
        return [data[off[i]:off[i + 1]] for i in range(2 * n)]

    b0, b2 = records(ws0), records(ws2)
    once = np.flatnonzero((o2["rounds"] == 1).all(axis=0))
    assert 0 < len(once) < n
    for i in once:
        assert b0[2 * i] == b2[2 * i] and b0[2 * i + 1] == b2[2 * i + 1], i


def test_arguments(world):
    w = world
    n = w["n_pairs"]
    rs = packed(w["reads"])
    p, pair = params_for(aln.LOCAL), pair_for(aln.LOCAL)
    mq, rp = tables(aln.LOCAL, 2)
    ws = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], rs, p, pair, rp, mapq=mq, traceback=True, hit_capacity=64 * rs.count)
    torch.cuda.synchronize()
    L_ = lib()
    s, rd = w["fmi"].struct(), rs.struct()
    tb = C.c_size_t(ws.temp_bytes)
    po = PairOutStruct()
    po.d_pair_score, po.d_pair_flags = ws.pair_score.data_ptr(), ws.pair_flags.data_ptr()
    po.d_mate_score, po.d_mate_pos, po.d_mate_strand = ws.mate_score.data_ptr(), ws.mate_pos.data_ptr(), ws.mate_strand.data_ptr()
    ro = ReseedOutStruct()
    ro.d_rounds, ro.d_active = ws.rounds.data_ptr(), ws.active.data_ptr()
    from nvbio_b200.pipeline import _p
    from nvbio_b200._lib import BestAlignmentOutStruct, PairMapqOutStruct
    ba = BestAlignmentOutStruct()
    ba.d_ops, ba.max_ops, ba.d_n_ops, ba.d_begin = ws.mate_ops.data_ptr(), ws.max_ops, ws.mate_n_ops.data_ptr(), ws.mate_begin.data_ptr()
    mo = PairMapqOutStruct()
    mo.d_second_pair_score, mo.d_mate_mapq = ws.second_pair_score.data_ptr(), ws.mate_mapq.data_ptr()
    mo.d_mate_second_score = ws.mate_second_score.data_ptr()             # (as the workspace's call: the same temp size)
    ref = lambda x: C.byref(x) if x is not None else None       # noqa: E731

    def call(rp_=rp.struct(), ps=p.struct(), pp=pair.struct(n), po_=po, ba_=None, mp=None, mo_=None, n_pairs=n, rd_=rd, ro_=ro):
        return L_.nvb_seed_extend_paired_reseed(C.byref(s), _p(w["gw"]), C.byref(rd_), C.c_uint32(n_pairs), C.byref(ps), C.c_uint32(64 * rs.count),
                                                ref(pp), ref(po_), ref(ba_), ref(mp), ref(mo_), ref(rp_), C.byref(ro_), None,
                                                _p(ws.temp), C.byref(tb), None)

    assert call() == 0 and call(ba_=ba, mp=mq.struct(), mo_=mo) == 0
    bad = rp.struct(); bad.d_min_score = None; bad.max_read_len = 0        # not read by the paired rule
    assert call(rp_=bad) == 0
    torch.cuda.synchronize()
    assert call(rp_=None) == -1
    bad = rp.struct(); bad.max_reseed = 255
    assert call(rp_=bad) == -1
    bad = rp.struct(); bad.max_reseed = 24                                 # seed_interval 24 < 25 rounds
    assert call(rp_=bad) == -1
    bad.max_reseed = 23
    assert call(rp_=bad, ro_=ReseedOutStruct()) == 0                       # (d_active holds 3 rounds: no reseed outputs)
    torch.cuda.synchronize()
    assert call(pp=None) == -1 and call(po_=None) == -1 and call(n_pairs=0x40000000) == -1
    ps = p.struct(); ps.both_strands = 0
    assert call(ps=ps) == -1
    for f in ("max_frag", "min_frag"):
        pp = pair.struct(n)
        if f == "max_frag":
            pp.max_frag = 0
        else:
            pp.min_frag = pp.max_frag + 1
        assert call(pp=pp) == -1, f
    bad_po = PairOutStruct(); C.memmove(C.addressof(bad_po), C.addressof(po), C.sizeof(po)); bad_po.d_mate_pos = None
    assert call(po_=bad_po) == -1
    assert call(mp=mq.struct()) == -1 and call(mo_=mo) == -1                  # only one of mapq / mapq_out
    long_rd = rs.struct(); long_rd.length = 513
    assert call(ba_=ba, rd_=long_rd) == -4
    # n_pairs == 0: OK, d_active zeroed
    ws.active.fill_(7)
    assert call(n_pairs=0) == 0
    torch.cuda.synchronize()
    assert ws.active.tolist() == [0, 0, 0]
