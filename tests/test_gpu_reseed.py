"""-m gpu: reseeding rounds of nvb_seed_extend_reseed against the round-by-round oracle (tests/reseed_oracle.py) on a genome with a
planted 16-copy repeat family: bit-identical to nvb_seed_extend[_traceback|_mapq] at max_reseed = 0, the oracle's rounds, active counts,
best / second / MAPQ and per-hit arrays on every path, nvb_map_seeds' own range statistics and flags, the traceback, the BAM chain and
the argument checks."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams, ReseedParams
from nvbio_b200.strings import PackedStringSet, pack_symbols
from nvbio_b200._lib import ReseedOutStruct
from tests.gpu_util import require_gpu, host_u32
from tests.reseed_oracle import seed_extend_reseed_oracle
from tests.mapq_oracle import INT_MIN

pytestmark = pytest.mark.gpu

G = 300_000
RL, L, I = 90, 16, 24          # with both strands, round 0's seeds of a 90 bp read leave [18, 24), [42, 48), [66, 72) uncovered
UNIT, COPIES = 300, 16
SUBST = [2, 26, 50, 74]        # covered by every round-0 seed of both strings, by no seed at offset 8 (max_reseed = 2, round 1)
N_SUB, N_REP, N_ORD = 60, 64, 200


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def world_data():
    rng = np.random.default_rng(11)
    g = rng.integers(0, 4, G).astype(np.uint8)
    unit = rng.integers(0, 4, UNIT).astype(np.uint8)
    starts = [5_000 + 17_000 * c for c in range(COPIES)]
    for c, st in enumerate(starts):
        u = unit.copy()
        u[30 + 15 * c] = (u[30 + 15 * c] + 1) % 4               # copy c's own variant
        g[st:st + UNIT] = u
    reads, truth = [], []
    for i in range(N_SUB):                                        # substitution reads: rescued only by shifted seeds
        p = 280_000 + 300 * i
        r = g[p:p + RL].copy()
        r[SUBST] = (r[SUBST] + 1 + rng.integers(0, 3, len(SUBST))) % 4
        if i % 2:
            r = rc(r)
        reads.append(r); truth.append(p)
    for i in range(N_REP):                                        # repeat reads: copy c's variant at read position 20
        c = i % COPIES
        p = starts[c] + 10 + 15 * c
        r = g[p:p + RL].copy()
        if i % 2:
            r = rc(r)
        reads.append(r); truth.append(p)
    for i in range(N_ORD):                                        # ordinary reads, some short, some mutated, some from nowhere
        ln = RL if i % 5 else int(rng.integers(14, RL))
        p = int(rng.integers(0, G - ln))
        r = g[p:p + ln].copy()
        if i % 3 == 1:
            m = rng.random(ln) < 0.06
            r[m] = (r[m] + 1) % 4
        if i % 17 == 0:
            r = rng.integers(0, 4, ln).astype(np.uint8)
        if i % 2:
            r = rc(r)
        reads.append(r); truth.append(p)
    return g, reads, np.array(truth)


@pytest.fixture(scope="module")
def world():
    require_gpu()
    O = orc.Oracle()
    g, reads, truth = world_data()
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    fmi_loc = nb.FMIndexDevice.from_text(gw, G, sa_interval=1)[0]
    fmi_loc.build_ktab(8, located=True, text=gw)
    return dict(O=O, g=g, gw=gw, idx=idx, fmi=fmi, fmi_loc=fmi_loc, reads=reads, truth=truth)


def packed(reads, bits=2):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = (np.cumsum(lens) - lens).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)
    rs.length = RL
    return rs


def params_for(typ, qual=None, both=True, hits=4):
    if qual is not None:
        sch = aln.QualityGotohScheme(2 if typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3)
    else:
        sch = aln.SimpleGotohScheme(2, -2, -5, -3) if typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
    return nb.SeedExtendParams(seed_len=L, seed_interval=I, band_len=15, type=typ, both_strands=both, max_seed_hits=hits, scheme=sch,
                               read_quals=qual)


def tables(typ, max_reseed, rep=8):
    mq = MapqParams.local(RL) if typ == aln.LOCAL else MapqParams.end_to_end(RL)
    return mq, ReseedParams(mq.min_score, max_reseed, rep)


KEYS = ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq")


def outs(ws):
    o = {}
    for k in KEYS:
        if getattr(ws, k) is not None:
            a = getattr(ws, k).cpu().numpy()
            o[k] = (a.view(np.uint32) if k in ("best_pos", "second_pos") else a).astype(np.int64)
    o["rounds"] = ws.rounds.cpu().numpy().astype(np.int64)
    o["active"] = ws.active.cpu().numpy().astype(np.int64)
    return o


def test_max_reseed_zero_is_seed_extend(world):
    """max_reseed = 0: every output bit-identical to nvb_seed_extend_mapq / _traceback / plain, on both paths"""
    w = world
    rs = packed(w["reads"])
    for typ in (aln.LOCAL, aln.SEMI_GLOBAL):
        p = params_for(typ)
        mq, rp = tables(typ, 0)
        for keep in (False, True):
            for fmi in (w["fmi"], w["fmi_loc"]):
                for tb, m in ((True, mq), (False, None), (True, None)):
                    a = nb.seed_extend(fmi, w["gw"], rs, p, hit_capacity=64 * rs.count, keep_hits=keep, traceback=tb, mapq=m)
                    b = nb.seed_extend_reseed(fmi, w["gw"], rs, p, rp, traceback=tb, mapq=m, keep_hits=keep, hit_capacity=64 * rs.count)
                    torch.cuda.synchronize()
                    for k in ("best_score", "best_pos", "n_hits", "hit_read", "hit_window", "hit_score", "hit_sink", "best_ops", "best_n_ops",
                              "best_begin", "best_strand", "second_score", "second_pos", "second_strand", "mapq"):
                        x, y = getattr(a, k), getattr(b, k)
                        assert (x is None) == (y is None), k
                        if x is not None:
                            n = int(a.n_hits[0]) if k.startswith("hit_") else x.shape[0]
                            assert torch.equal(x[:n], y[:n]), (typ, keep, tb, k)
                    assert (b.rounds == 1).all() and b.active.tolist() == [rs.count]


CONFIGS = [(2, aln.LOCAL, False), (4, aln.LOCAL, False), (2, aln.SEMI_GLOBAL, False), (2, aln.LOCAL, True)]


@pytest.mark.parametrize("max_reseed", [1, 2, 3])
@pytest.mark.parametrize("bits,typ,qual", CONFIGS)
def test_vs_oracle(world, max_reseed, bits, typ, qual):
    w = world
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        rng = np.random.default_rng(5)
        for r in reads[N_SUB + N_REP::7]:
            r[rng.integers(0, len(r), 1)] = 4                     # N
    quals = None
    qt = None
    if qual:
        rng = np.random.default_rng(9)
        quals = [rng.integers(0, 45, len(r)).astype(np.uint8) for r in reads]
        qt = torch.from_numpy(np.concatenate(quals)).cuda()
    rs = packed(reads, bits)
    p = params_for(typ, qt)
    mq, rp = tables(typ, max_reseed)
    cap = 64 * rs.count
    want = seed_extend_reseed_oracle(w["O"], w["idx"], w["g"], reads, p, max_reseed, 8, mq.min_score.cpu().numpy(), cap,
                                     match_bonus=mq.match_bonus, quals=quals)
    assert want["active"][1] > N_SUB and want["active"][0] == len(reads)

    def check(ws, what):
        got = outs(ws)
        for k in got:
            bad = np.nonzero(got[k] != want[k])[0]
            assert len(bad) == 0, (what, k, [(int(i), int(got[k][i]), int(want[k][i])) for i in bad[:5]])
        assert host_u32(ws.n_hits)[:2].tolist() == list(want["n_hits"]), what

    L_ = nb.lib()
    # per-read path (default), both index formats, the exact shortcut at 0 / 1 / 2, the seed split off
    for fmi in (w["fmi"], w["fmi_loc"]):
        check(nb.seed_extend_reseed(fmi, w["gw"], rs, p, rp, traceback=True, mapq=mq, hit_capacity=cap), "per-read")
    for hook, val, dflt in ((L_.nvb_debug_perfect_shortcut, 0, 1), (L_.nvb_debug_perfect_shortcut, 2, 1), (L_.nvb_debug_seed_split, 0, 1)):
        hook(C.c_int(val))
        try:
            check(nb.seed_extend_reseed(w["fmi_loc"], w["gw"], rs, p, rp, mapq=mq, hit_capacity=cap), (hook.__name__, val))
        finally:
            hook(C.c_int(dflt))
    # per-hit path: the hit arrays hit by hit; with and without de-duplication
    for dedup in (True, False):
        p.dedup_jobs = dedup
        ws = nb.seed_extend_reseed(w["fmi"], w["gw"], rs, p, rp, mapq=mq, keep_hits=True, hit_capacity=cap)
        check(ws, ("per-hit", dedup))
        n = int(ws.n_hits[0])
        assert np.array_equal(ws.hit_read[:n].cpu().numpy(), want["hit_string"])
        assert np.array_equal(host_u32(ws.hit_window[:n]).astype(np.int64), want["hit_window"])
        assert np.array_equal(ws.hit_score[:n].cpu().numpy(), want["hit_score"])
        assert np.array_equal(host_u32(ws.hit_sink[:n]).astype(np.int64), want["hit_sink"])
    p.dedup_jobs = True


def test_capacity_overflows_in_round_one(world):
    w = world
    rs = packed(w["reads"])
    p = params_for(aln.LOCAL)
    mq, rp = tables(aln.LOCAL, 2)
    ws0 = nb.seed_extend(w["fmi"], w["gw"], rs, p, keep_hits=True, hit_capacity=64 * rs.count)
    cap = int(ws0.n_hits[0]) + 40
    want = seed_extend_reseed_oracle(w["O"], w["idx"], w["g"], w["reads"], p, 2, 8, mq.min_score.cpu().numpy(), cap, match_bonus=mq.match_bonus)
    assert want["n_hits"][0] == cap and want["n_hits"][1] > cap
    for keep in (True, False):
        ws = nb.seed_extend_reseed(w["fmi"], w["gw"], rs, p, rp, mapq=mq, keep_hits=keep, hit_capacity=cap)
        got = outs(ws)
        for k in got:
            assert np.array_equal(got[k], want[k]), (keep, k)
        if keep:
            assert np.array_equal(ws.hit_read.cpu().numpy(), want["hit_string"])
            assert np.array_equal(ws.hit_score.cpu().numpy(), want["hit_score"])


@pytest.mark.parametrize("max_reseed", [1, 2, 3])
def test_rule_is_map_seeds(world, max_reseed):
    """forward strand only: the oracle's per-round range statistics and flags are nvb_map_seeds' (EXACT, retry = r, seed_freq = I)"""
    w = world
    reads = [r for r in w["reads"] if len(r) >= L]
    p = params_for(aln.LOCAL, both=False)
    mq, _ = tables(aln.LOCAL, max_reseed)
    want = seed_extend_reseed_oracle(w["O"], w["idx"], w["g"], reads, p, max_reseed, 8, mq.min_score.cpu().numpy(), 10**9)
    rs = packed(reads)
    # nvBowtie seeds against the index of the reversed genome: a range's size is the same as the forward seed's on the forward index
    ridx = w["O"].build_index(np.ascontiguousarray(w["g"][::-1]))
    fmi_rev = nb.FMIndexDevice.from_host(ridx.bwt_occ, ridx.ssa, ridx.L2, ridx.n, ridx.primary)
    for r, st in enumerate(want["stats"]):
        q = np.array(sorted(st), np.int32)
        _, _, flag, stats = nb.map_seeds(fmi_rev, rs, nb.MAP_EXACT, seed_len=L, seed_freq=I, max_hits=64, max_reseed=max_reseed, rep_seeds=8,
                                         min_read_len=0, fw=True, rc=False, queue=torch.from_numpy(q).cuda(), retry=r)
        s = host_u32(stats).astype(np.int64)
        assert [tuple(s[i]) for i in range(len(q))] == [st[int(x)] for x in q], r
        if r < max_reseed:
            range_only = [int(st[int(x)][1] == 0 or st[int(x)][0] >= 8 * st[int(x)][1]) for x in q]
            assert flag.cpu().numpy().tolist() == range_only, r


def test_traceback_and_bam_chain(world):
    w = world
    reads = w["reads"]
    rs = packed(reads)
    p = params_for(aln.LOCAL)
    mq, rp0 = tables(aln.LOCAL, 0)
    _, rp2 = tables(aln.LOCAL, 2)
    ws0 = nb.seed_extend_reseed(w["fmi"], w["gw"], rs, p, rp0, traceback=True, mapq=mq)
    ws2 = nb.seed_extend_reseed(w["fmi"], w["gw"], rs, p, rp2, traceback=True, mapq=mq)
    torch.cuda.synchronize()
    # reads seeded once keep nvb_seed_extend_traceback's alignment; every alignment replays to its score and end
    rounds = ws2.rounds.cpu().numpy()
    one = rounds == 1
    for k in ("best_ops", "best_n_ops", "best_begin", "best_strand", "best_score", "best_pos", "mapq"):
        assert torch.equal(getattr(ws0, k)[torch.from_numpy(one).cuda()], getattr(ws2, k)[torch.from_numpy(one).cuda()]), k
    n_ops = ws2.best_n_ops.cpu().numpy()
    sc2 = ws2.best_score.cpu().numpy()
    assert ((sc2 != INT_MIN) == (n_ops > 0)).all()
    # ops replay to the score (LOCAL 2 / -2 / gap open 5, ext 3: a gap of k costs 5 + 3 (k - 1))
    g = w["g"]
    begin = host_u32(ws2.best_begin).astype(np.int64)
    strand = ws2.best_strand.cpu().numpy()
    ops = ws2.best_ops.cpu().numpy()
    for r in np.nonzero(n_ops > 0)[0]:
        s = reads[r] if strand[r] == 0 else rc(reads[r])
        seq = ops[r, :n_ops[r]][::-1]
        t, q, score, prev = begin[r, 0], begin[r, 1], 0, -1
        for o in seq:
            if o == 0:
                score += 2 if s[q] == g[t] else -2; q += 1; t += 1
            elif o == 1:
                score -= 5 if prev != 1 else 3; q += 1
            else:
                score -= 5 if prev != 2 else 3; t += 1
            prev = o
        assert score == sc2[r] and t == host_u32(ws2.best_pos)[r], r
    # the BAM chain on the reseeded workspace
    contigs = nb.ContigTable(["chr1"], [G])
    names = nb.numbered_names(len(reads))

    def records(ws):
        f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=G)
        recs = nb.bam_records(ws, f, rs, contigs, names)
        off = recs.offsets.cpu().numpy()
        data = recs.to_bytes()
        return [data[off[i]:off[i + 1]] for i in range(len(reads))]

    b0, b2 = records(ws0), records(ws2)
    assert all(b0[i] == b2[i] for i in np.nonzero(one)[0])
    flag = lambda rec: int.from_bytes(rec[18:20], "little")        # noqa: E731
    pos = lambda rec: int.from_bytes(rec[8:12], "little", signed=True)   # noqa: E731
    rescued = 0
    for i in range(N_SUB):
        assert flag(b0[i]) & 4, i                                  # unmapped without reseeding
        if not flag(b2[i]) & 4:
            assert abs(pos(b2[i]) - int(w["truth"][i])) <= 4, i
            rescued += 1
    assert rescued == N_SUB
    rep = slice(N_SUB, N_SUB + N_REP)
    true_end = w["truth"][rep] + RL
    moved = host_u32(ws2.best_pos)[rep].astype(np.int64) == true_end
    assert moved.all() and (host_u32(ws0.best_pos)[rep].astype(np.int64) != true_end).sum() > 0


def test_invalid_arguments(world):
    w = world
    rs = packed(w["reads"])
    p = params_for(aln.LOCAL)
    mq, rp = tables(aln.LOCAL, 2)
    ws = nb.seed_extend_reseed(w["fmi"], w["gw"], rs, p, rp, hit_capacity=1000)
    L_ = nb.lib()
    s, rd, ps = w["fmi"].struct(), rs.struct(), p.struct()
    tb = C.c_size_t(ws.temp_bytes)
    ro = ReseedOutStruct()

    def call(rp_struct, ps_struct=ps):
        return L_.nvb_seed_extend_reseed(C.byref(s), C.c_void_p(w["gw"].data_ptr()), C.byref(rd), C.c_uint32(rs.count), C.byref(ps_struct),
                                         C.c_uint32(1000), C.c_void_p(ws.best_score.data_ptr()), C.c_void_p(ws.best_pos.data_ptr()), None,
                                         None, None, None, None, None, None, None,
                                         C.byref(rp_struct) if rp_struct is not None else None, C.byref(ro),
                                         C.c_void_p(ws.temp.data_ptr()), C.byref(tb), None)

    good = rp.struct()
    assert call(good) == 0
    assert call(None) == -1
    bad = rp.struct(); bad.d_min_score = None
    assert call(bad) == -1
    bad = ReseedParams(mq.min_score[:RL], 2, 8).struct()           # table shorter than the reads
    assert call(bad) == -1
    bad = rp.struct(); bad.max_reseed = 255
    assert call(bad) == -1
    bad = rp.struct(); bad.max_reseed = 24                        # seed_interval 24 < 25 rounds
    assert call(bad) == -1
    bad.max_reseed = 23
    assert call(bad) == 0
    torch.cuda.synchronize()
