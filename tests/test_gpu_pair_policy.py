"""-m gpu: paired-end seed + extend under every pairing policy and option (nvb_pair_params.policy / flags): FR, RF, FF and RR, with and
without overlap, discordant pairs and --no-mixed.  The outputs of the paired calls equal the oracle composition extended by the policy
(tests/pair_policy_oracle.py) on both extension paths, with and without job
de-duplication and under a quality scheme; rescued mates' tracebacks equal nvb_gotoh_traceback of the rebuilt job; discordant and
--no-mixed pairs carry the outputs the header states, down to the BAM flags; pairs generated in each orientation pair up under their
policy; the reseeding call and the streaming pipeline follow the policy."""
from unittest import mock
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.pipeline import MapqParams, ReseedParams
from nvbio_b200.strings import PackedStringSet
from tests import pipeline_oracle, pair_policy_oracle as ppo
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import seed_extend_oracle
from tests.pair_policy_oracle import rescue_window, seed_extend_paired_reseed_oracle
from tests.test_gpu_paired_traceback import strand_string, replay

INT_MIN = -2**31
NONE = 0xFFFFFFFF
RL, G, UNIT, COPIES = 100, 300_000, 700, 8
POLICIES = ("fr", "rf", "ff", "rr")
CLASSES = ("clean", "rescue", "elsewhere", "family", "overlap", "long")
PAIR_KEYS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue")
MAPQ_KEYS = ("second_pair_score", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")
TB_KEYS = ("mate_ops", "mate_n_ops", "mate_begin")


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def orient(g, left, frag, orientation, odd):
    """(mate 1, mate 2) of the fragment [left, left + frag) sequenced in `orientation` (synth.sample_pairs' table)"""
    seg = dict(fwL=g[left:left + RL].copy(), fwR=g[left + frag - RL:left + frag].copy())
    seg["rvL"], seg["rvR"] = rc(seg["fwL"]), rc(seg["fwR"])
    a, b = synth._ORIENT[orientation][1 if odd else 0]
    return seg[a], seg[b]


def make_world(per_class=(10, 6, 6, 6, 5, 5), seed=41):
    """genome with a planted COPIES-copy family; pairs of every class in every orientation.  cls[p], orient[p]; mate 1s then mate 2s"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, G).astype(np.uint8)
    unit = rng.integers(0, 4, UNIT).astype(np.uint8)
    starts = [200_000 + 11_000 * c for c in range(COPIES)]
    for st in starts:
        g[st:st + UNIT] = unit
    m1, m2, cls, ori = [], [], [], []
    for oi, o in enumerate(POLICIES):
        for ci, n in enumerate(per_class):
            for i in range(n):
                name = CLASSES[ci]
                frag = int(rng.integers(200, 400))
                left = int(rng.integers(1_000, 190_000 - 1_000))
                if name == "family":
                    left, frag = starts[i % COPIES] + int(rng.integers(0, UNIT - 400)), int(rng.integers(250, 400))
                elif name == "overlap":
                    frag = int(rng.integers(RL, RL + 60))
                elif name == "long":
                    frag = int(rng.integers(600, 900))
                a, b = orient(g, left, frag, o, i % 2 == 1)
                if name == "rescue":                                # mate 2 heavily substituted: no exact seed, the rescue places it
                    mm = rng.random(RL) < 0.2
                    b[mm] = (b[mm] + 1) % 4
                elif name == "elsewhere":                           # mate 2 from another locus, either strand
                    q = int(rng.integers(1_000, 190_000 - 1_000))
                    b = g[q:q + RL].copy() if rng.random() < 0.5 else rc(g[q:q + RL])
                else:
                    for r in (a, b):
                        mm = rng.random(RL) < 0.01
                        r[mm] = (r[mm] + 1) % 4
                m1.append(a); m2.append(b); cls.append(ci); ori.append(oi)
    return g, m1 + m2, np.array(cls), np.array(ori)


@pytest.fixture(scope="module")
def world():
    require_gpu()
    O = orc.Oracle()
    g, reads, cls, ori = make_world()
    gw = torch.from_numpy(nb.pack_symbols(g, bits=2, big_endian=True, pad_words=8).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    rng = np.random.default_rng(9)
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    return dict(O=O, g=g, gw=gw, idx=idx, fmi=fmi, reads=reads, quals=quals, cls=cls, ori=ori, n_pairs=len(cls), se={})


def read_set(w):
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    return PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=2, big_endian=True)


def make_params(w=None, qual=False, dedup=True):
    if qual:
        return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                                   dedup_jobs=dedup, scheme=aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3),
                                   read_quals=torch.from_numpy(np.concatenate(w["quals"])).cuda())
    return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                               dedup_jobs=dedup, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


_MQ = []


def mq():
    """the MAPQ inputs of every call here (made on first use: the device is needed)"""
    if not _MQ:
        _MQ.append(MapqParams.local(RL))
    return _MQ[0]


def run(w, pair, qual=False, dedup=True, mapq=True, traceback=False, path=None):
    mapq = mq() if mapq else None
    if path is not None:
        nb.lib().nvb_debug_pipeline_path(path)
    try:
        ws = nb.seed_extend_paired(w["fmi"], w["gw"], read_set(w), make_params(w, qual, dedup), pair, hit_capacity=64 * 2 * w["n_pairs"],
                                   mapq=mapq, traceback=traceback)
        torch.cuda.synchronize()
    finally:
        if path is not None:
            nb.lib().nvb_debug_pipeline_path(0)
    keys = PAIR_KEYS + (MAPQ_KEYS if mapq is not None else ()) + (TB_KEYS if traceback else ())
    return {k: getattr(ws, k).cpu().numpy().copy() for k in keys}, ws


def oracle(w, pair, qual=False, mapq=True):
    """the oracle composition under pair's policy; the single-end stage (the same for every policy) is computed once per scheme"""
    params = make_params(w, qual)
    if qual not in w["se"]:
        w["se"][qual] = seed_extend_oracle(w["O"], w["idx"], w["g"], w["reads"], params, quals=w["quals"] if qual else None)
    se = w["se"][qual]
    cached = lambda *a, **k: se                                            # noqa: E731
    q = w["quals"] if qual else None
    with mock.patch.object(pipeline_oracle, "seed_extend_oracle", cached):
        if mapq:
            return ppo.pair_mapq_oracle(w["O"], w["idx"], w["g"], w["reads"], params, pair, w["n_pairs"], mq().min_score.cpu().numpy(), mq().match_bonus,
                                        quals=q)
        return ppo.seed_extend_paired_oracle(w["O"], w["idx"], w["g"], w["reads"], params, pair, w["n_pairs"], quals=q)


def compare(got, want, keys):
    for k in keys:
        g = got[k].astype(np.int64)
        wv = np.asarray(want[k], np.int64).reshape(g.shape)
        if k in ("mate_pos", "second_mate_pos"):                            # device outputs are int32 views of uint32
            g, wv = g & 0xFFFFFFFF, wv & 0xFFFFFFFF
        bad = np.argwhere(g != wv)
        assert len(bad) == 0, (k, bad[:5].tolist(), g[tuple(bad[0])], wv[tuple(bad[0])])


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("overlap", [True, False])
def test_policy_vs_oracle(world, policy, overlap):
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy=policy, overlap=overlap)
    want = oracle(w, pair)
    got, _ = run(w, pair)
    compare(got, want, PAIR_KEYS + MAPQ_KEYS)
    plain, _ = run(w, pair, mapq=False)
    compare(plain, want, PAIR_KEYS)
    for variant in (dict(path=1), dict(dedup=False)):                     # the per-hit path; no de-duplication
        compare(run(w, pair, **variant)[0], want, PAIR_KEYS + MAPQ_KEYS)
    tb, _ = run(w, pair, traceback=True)
    compare(tb, want, PAIR_KEYS + MAPQ_KEYS)
    flags = got["pair_flags"]
    mine = w["ori"] == POLICIES.index(policy)
    assert (flags[mine] == 1).sum() > 0 and ((flags == 2) | (flags == 4)).sum() > 0


@pytest.mark.gpu
def test_policy_quality_scheme_vs_oracle(world):
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=50, policy="rr", overlap=False, discordant=True, mixed=False)
    want = oracle(w, pair, qual=True)
    compare(run(w, pair, qual=True)[0], want, PAIR_KEYS + MAPQ_KEYS)
    compare(run(w, pair, qual=True, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS)


@pytest.mark.gpu
@pytest.mark.parametrize("mixed", [True, False])
def test_discordant_pairs(world, mixed):
    w = world
    n = w["n_pairs"]
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy="fr", discordant=True, mixed=mixed)
    want = oracle(w, pair)
    got, ws = run(w, pair, traceback=True)
    compare(got, want, PAIR_KEYS + MAPQ_KEYS)
    flags = got["pair_flags"]
    disc = flags == nb.PAIR_DISCORDANT
    assert disc.sum() >= 10
    assert not disc[w["cls"] == CLASSES.index("family")].any()               # repeat-family mates are never unique
    assert disc[(w["cls"] == CLASSES.index("elsewhere")) & (w["ori"] == 0)].sum() >= 3
    # the rules of the header: s1 + s2, no second pair, MAPQ of the pair score without a second
    ms = mq().min_score.cpu().numpy()
    for p in np.flatnonzero(disc):
        s1, s2 = int(got["mate_score"][0, p]), int(got["mate_score"][1, p])
        assert got["pair_score"][p] == s1 + s2 and got["second_pair_score"][p] == INT_MIN
        assert (got["second_mate_pos"][:, p].astype(np.uint32) == NONE).all() and (got["second_mate_strand"][:, p] == 0).all()
        assert (got["mate_second_score"][:, p] == INT_MIN).all()
        q = ppo.bowtie_mapq2(s1 + s2, False, 0, 2 * RL, mq().match_bonus, 2 * int(ms[RL]))
        assert (got["mate_mapq"][:, p] == q).all()
    un = flags == nb.PAIR_UNPAIRED
    if not mixed:
        assert un.sum() > 0
        assert (got["mate_score"][:, un] == INT_MIN).all() and (got["mate_pos"][:, un].astype(np.uint32) == NONE).all()
        assert (got["mate_strand"][:, un] == 0).all() and (got["mate_mapq"][:, un] == 0).all()
        assert (got["mate_second_score"][:, un] == INT_MIN).all()
        assert (got["mate_n_ops"][:, un] == 0).all() and (got["mate_begin"][:, un].view(np.uint32) == NONE).all()
    # BAM: 0x2 only on CONCORDANT / RESCUED pairs; a discordant record carries 0x1, 0x40 / 0x80 and the mate fields without 0x2
    rs = read_set(w)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    contigs = nb.ContigTable(["chrA", "chrB"], [G // 2, G - G // 2])
    recs = nb.bam_records(ws, f, rs, contigs, nb.numbered_names(n, "pair"))
    torch.cuda.synchronize()
    off, data = recs.offsets.cpu().numpy(), recs.data.cpu().numpy()
    seen_disc = 0
    for p in range(n):
        for m in range(2):
            rec = data[off[2 * p + m]:off[2 * p + m + 1]]
            flag = int(rec[18]) | int(rec[19]) << 8                            # bam1_t: flag_nc = block_size, refID, pos, l_read_name/mapq/bin, flag
            assert flag & 0x1 and flag & (0x80 if m else 0x40)
            mapped = got["mate_pos"][m, p].astype(np.uint32) != NONE
            proper = flags[p] in (1, 2, 4)
            if not (flag & 0x4) and not (flag & 0x8):
                assert bool(flag & 0x2) == proper, (p, m, flag, flags[p])
            if disc[p] and not (flag & 0x4) and not (flag & 0x8):
                seen_disc += 1
                assert not flag & 0x2
                nref, npos = (int(v) for v in np.frombuffer(rec[24:32].tobytes(), np.int32))
                assert nref >= 0 and npos >= 0
            if not mixed and un[p]:
                assert flag & 0x4 and flag & 0x8 and not mapped
    assert seen_disc > 0
    sam = nb.sam_text(recs, contigs)
    torch.cuda.synchronize()
    so, sd = sam.offsets.cpu().numpy(), sam.data.cpu().numpy().tobytes()
    assert int(sam.rejected[0]) == 0
    for i in range(2 * n):
        line = sd[so[i]:so[i + 1]].decode()
        assert line.endswith("\n") and len(line.rstrip("\n").split("\t")) >= 11, line
        fl = int(line.split("\t")[1])
        p = i // 2
        if disc[p] and not fl & 0xC:
            assert fl & 0x1 and not fl & 0x2


@pytest.mark.gpu
def test_traceback_under_policy(world):
    """pair and MAPQ outputs as _paired_mapq; mates that keep their single-end best: the single-end traceback; rescued mates: the full
    traceback of the rebuilt job (rescue window and strand of the policy); --no-mixed mates: unaligned; every aligned mate replays"""
    w = world
    n, reads = w["n_pairs"], w["reads"]
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy="rf", overlap=False, discordant=True, mixed=False)
    got, ws = run(w, pair, traceback=True)
    ref, _ = run(w, pair)
    compare(got, ref, PAIR_KEYS + MAPQ_KEYS)
    params = make_params(w)
    se = nb.seed_extend(w["fmi"], w["gw"], read_set(w), params, hit_capacity=64 * 2 * n, traceback=True)
    torch.cuda.synchronize()
    se_ops, se_n, se_begin = se.best_ops.cpu().numpy(), se.best_n_ops.cpu().numpy(), host_u32(se.best_begin)
    se_pos, se_strand = host_u32(se.best_pos), se.best_strand.cpu().numpy()
    flags, mops, mn, mbeg = got["pair_flags"], got["mate_ops"], got["mate_n_ops"], got["mate_begin"].view(np.uint32)
    rescued = []
    for p in range(n):
        for m in range(2):
            r = m * n + p
            if flags[p] in (2, 4) and m == (0 if flags[p] == 2 else 1):
                rescued.append((p, m)); continue
            if flags[p] == 0:
                assert mn[m, p] == 0 and tuple(mbeg[m, p]) == (NONE, NONE); continue
            assert mn[m, p] == se_n[r] and np.array_equal(mbeg[m, p], se_begin[r]), (p, m)
            assert np.array_equal(mops[m, p, :mn[m, p]], se_ops[r, :se_n[r]]), (p, m)
    assert len(rescued) >= 3
    pats, t_off, t_len = [], [], []
    for p, o in rescued:
        a = 1 - o
        ra, ro = a * n + p, o * n + p
        end = int(se_pos[ra])
        to, te, ot = rescue_window("rf", False, a, int(se_strand[ra]), max(end - len(reads[ra]), 0), end, pair.max_frag, G)
        assert got["mate_strand"][o, p] == ot
        pats.append(strand_string(reads[ro], w["quals"][ro], ot)[0]); t_off.append(to); t_len.append(te - to)
    lens = np.array([len(x) for x in pats], np.uint32)
    P = PackedStringSet.from_symbols(np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, bits=2)
    T = PackedStringSet.from_symbols(w["g"], np.array(t_off, np.uint32), np.array(t_len, np.uint32), bits=2)
    want = aln.batch_alignment_traceback(aln.make_gotoh_aligner(aln.LOCAL, params.scheme), P, T, max_ops=ws.max_ops)
    torch.cuda.synchronize()
    ws_ops, ws_n, ws_src, ws_sink = want["ops"].cpu().numpy(), host_u32(want["n_ops"]), host_u32(want["source"]), host_u32(want["sink"])
    for i, (p, o) in enumerate(rescued):
        assert int(want["score"][i]) == got["mate_score"][o, p] and t_off[i] + ws_sink[i][0] == np.uint32(got["mate_pos"][o, p])
        assert mn[o, p] == ws_n[i] and tuple(mbeg[o, p]) == (t_off[i] + ws_src[i][0], ws_src[i][1]), (p, o)
        assert np.array_equal(mops[o, p, :ws_n[i]], ws_ops[i, :ws_n[i]]), (p, o)
    for p in range(n):
        for m in range(2):
            if np.uint32(got["mate_pos"][m, p]) == NONE:
                continue
            r = m * n + p
            pat, q = strand_string(reads[r], w["quals"][r], int(got["mate_strand"][m, p]))
            assert replay(mops[m, p], mn[m, p], mbeg[m, p], pat, q, w["g"], params.scheme) == (int(got["mate_score"][m, p]),
                                                                                                 int(got["mate_pos"][m, p])), (p, m)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_orientation_sanity(policy):
    """pairs generated in orientation X pair up under policy X (>= 99 % concordant or rescued, both mates within 20 bp of the truth);
    FR pairs longer than a read are never CONCORDANT under RF"""
    require_gpu()
    n, n_pairs = 400_000, 4000
    gw = synth.random_genome_words(n, seed=5)
    fmi, _ = nb.FMIndexDevice.from_text(gw, n)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                                 scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy=policy)
    rw, left, frag = synth.sample_pairs(gw, n, n_pairs, RL, frag_mean=300, frag_sd=30, sub_rate=0.005, hard_frac=0.0, orientation=policy)
    rs = PackedStringSet.fixed(rw.reshape(-1), 2 * n_pairs, RL, stride=rw.shape[1] * 16)
    ws = nb.seed_extend_paired(fmi, gw, rs, params, pair, hit_capacity=64 * 2 * n_pairs)
    torch.cuda.synchronize()
    flags, pos = ws.pair_flags.cpu().numpy(), host_u32(ws.mate_pos)
    left, frag = left.cpu().numpy(), frag.cpu().numpy()
    ok = np.isin(flags, (1, 2, 4))
    assert ok.mean() >= 0.99, ok.mean()
    end = dict(L=left + RL, R=left + frag)
    for odd in (0, 1):
        sel = ok & (np.arange(n_pairs) % 2 == odd)
        for m in range(2):
            seg = synth._ORIENT[policy][odd][m][2]
            assert (np.abs(pos[m][sel].astype(np.int64) - end[seg][sel]) <= 20).all(), (policy, odd, m)
    if policy == "fr":
        rf = nb.seed_extend_paired(fmi, gw, rs, params, nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy="rf"),
                                   hit_capacity=64 * 2 * n_pairs)
        torch.cuda.synchronize()
        f2 = rf.pair_flags.cpu().numpy()
        assert not ((f2 == 1) & (frag > RL)).any()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", ("rf", "ff", "rr"))
def test_reseed_under_policy(world, policy):
    w = world
    n = w["n_pairs"]
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy=policy, overlap=policy != "ff", discordant=True,
                         mixed=policy != "rr")
    base, _ = run(w, pair)
    cap = 64 * 2 * n
    ws = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], read_set(w), make_params(w), pair, ReseedParams(mq().min_score, max_reseed=0, rep_seeds=300),
                                      mapq=mq(), hit_capacity=cap)
    torch.cuda.synchronize()
    compare({k: getattr(ws, k).cpu().numpy() for k in PAIR_KEYS + MAPQ_KEYS}, base, PAIR_KEYS + MAPQ_KEYS)
    if policy == "rr":
        ws2 = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], read_set(w), make_params(w), pair, ReseedParams(mq().min_score, max_reseed=2, rep_seeds=3),
                                           mapq=mq(), hit_capacity=cap)
        torch.cuda.synchronize()
        want = seed_extend_paired_reseed_oracle(w["O"], w["idx"], w["g"], w["reads"], make_params(w), pair, n, 2, 3, cap,
                                                min_score=mq().min_score.cpu().numpy(), match_bonus=mq().match_bonus)
        compare({k: getattr(ws2, k).cpu().numpy() for k in PAIR_KEYS + MAPQ_KEYS}, want, PAIR_KEYS + MAPQ_KEYS)
        assert (ws2.rounds.cpu().numpy() > 1).any()


@pytest.mark.gpu
def test_streaming_pipeline_under_policy():
    """nvb_pipeline under RF + no overlap + no mixed equals seed_extend_paired"""
    require_gpu()
    n, n_pairs = 200_000, 2000
    gw = synth.random_genome_words(n, seed=8)
    fmi, _ = nb.FMIndexDevice.from_text(gw, n)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                                 scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=60, policy="rf", overlap=False, mixed=False)
    rw, _, _ = synth.sample_pairs(gw, n, n_pairs, RL, frag_mean=250, frag_sd=60, orientation="rf", seed=3, mut_seed=4)
    rs = PackedStringSet.fixed(rw.reshape(-1), 2 * n_pairs, RL, stride=rw.shape[1] * 16)
    want = nb.seed_extend_paired(fmi, gw, rs, params, pair, hit_capacity=24 * 2 * n_pairs)
    torch.cuda.synchronize()
    st = nb.StreamingSeedExtend(fmi, gw, params, 2 * n_pairs, RL, rw.shape[1], hit_capacity=24 * 2 * n_pairs, depth=2, pair=pair)
    host = rw.cpu().pin_memory()
    got = st.result(st.submit(host))
    for k in ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand"):
        v = getattr(want, k).cpu()
        assert torch.equal(got[k].reshape(v.shape), v), k
    flags = want.pair_flags.cpu().numpy()
    assert (flags == 0).sum() > 0 and (flags == 1).sum() > 0.6 * n_pairs
    with pytest.raises(nb.NvbError):
        nb.StreamingSeedExtend(fmi, gw, params, 2 * n_pairs, RL, rw.shape[1], hit_capacity=1024, depth=2,
                               pair=nb.PairParams(policy="rf", discordant=True))
