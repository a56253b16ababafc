"""-m gpu: paired-end seed + extend under every pairing policy at its fragment, mate-length and genome edges.  tests/test_gpu_pair_policy.py
runs the policies on sampled pairs in the middle of a genome, 100 bp, 2-bit, min_frag 0; here the pairs are planted where the paired
kernels can go wrong, in every orientation and with either mate first:

  * fragments starting within 30 bp of position 0 and ending within 30 bp of the genome's end, the mate nearest the end heavily
    substituted, so that the other mate anchors a rescue window clipped at 0 (a left window) or at the genome's length (a right one);
  * exact mates on fragments of min_frag - 1, min_frag, max_frag and max_frag + 1, and rescued mates on fragments below min_frag (the
    rescue window ignores min_frag);
  * mates of unequal length (33 to 250 bp), and a 505-512 bp mate, longer than max_frag, whose --no-overlap window is empty;
  * 4-bit mates with N, rescued with their N reversed and complemented;
  * a four-copy repeat family (second pairs), and mates of two far-apart loci (discordant pairs).

Every policy x overlap x min_frag in {0, 200}: nvb_seed_extend_paired and _paired_mapq against the policy oracle
(tests/pair_policy_oracle.py) on the per-read and per-hit paths, with and without job de-duplication, and a rescue_capacity that cuts the
job list; then discordant pairs (with and without --no-mixed) traced by _paired_traceback: mates that keep their single-end best equal
the single-end traceback, rescued mates equal nvb_gotoh_traceback of the policy's window, every mate replays to its score and end; and
finish -> bam_records -> sam_text equal tests/bam_oracle.py and tests/sam_oracle.py byte for byte.  The quality scheme under every
policy; long mates (300-512 bp) under RF and FF.  Every planted edge is counted per configuration and must have happened."""
from unittest import mock
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet
from tests import pipeline_oracle, pair_policy_oracle as ppo, bam_oracle, sam_oracle
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import seed_extend_oracle, best_hits
from tests.test_gpu_paired_traceback import strand_string, replay, PAIR_KEYS, MAPQ_KEYS, TB_KEYS

INT_MIN = -2**31
NONE = 0xFFFFFFFF
G = 200_003
MAXF, MINF = 500, 200
UNIT = 800
FAMILY = (80_000, 105_000, 130_000, 155_000)
POLICIES = ("fr", "rf", "ff", "rr")
SEED_LEN, SEED_INTERVAL, MAX_SEED_HITS = 20, 10, 50
MAX_LEN = 512


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def mutate(r, rate, rng):
    r = r.copy()
    m = rng.random(len(r)) < rate
    r[m] = (r[m] + 1 + rng.integers(0, 3, int(m.sum()))) % 4
    return r


def mates(g, o, odd, left, frag, lens):
    """(mate 1, mate 2) of the fragment [left, left + frag) read in orientation o (synth._ORIENT, odd pairs off the other strand), mate
    m lens[m] long; and which mate is the fragment's left one"""
    out, left_mate = [], 0
    for m, seg in enumerate(synth._ORIENT[o][odd]):
        ln = lens[m]
        s = g[left:left + ln] if seg[2] == "L" else g[left + frag - ln:left + frag]
        out.append(rc(s) if seg[:2] == "rv" else s.copy())
        if seg[2] == "L":
            left_mate = m
    return out, left_mate


def plant(g, rng, long_mates=False):
    """(reads: mate 1s then mate 2s, kind of every pair, fragment of every pair (0: none)) for every orientation and parity"""
    m1, m2, kind, frags = [], [], [], []

    def add(o, odd, left, frag, lens, k, hard=None, rate=0.01, n_rate=0.0):
        (a, b), lm = mates(g, o, odd, left, frag, lens)
        pair = [mutate(a, rate, rng), mutate(b, rate, rng)]
        if hard is not None:                                     # that mate ("left" / "right" one, or mate 0 / 1) heavily substituted
            h = {"left": lm, "right": 1 - lm}.get(hard, hard)
            pair[h] = mutate(pair[h], 0.2, rng)
        for r in pair:
            r[rng.random(len(r)) < n_rate] = 4
        m1.append(pair[0]); m2.append(pair[1]); kind.append(k); frags.append(frag)

    for o in POLICIES:
        for odd in (0, 1):
            if long_mates:
                for _ in range(6):
                    lens = [int(x) for x in rng.integers(300, MAX_LEN + 1, 2)]
                    frag = int(rng.integers(max(lens) + 50, 1_150))
                    add(o, odd, int(rng.integers(1_000, G - 2_000)), frag, lens, "plain", rate=0.005)
                    add(o, odd, int(rng.integers(1_000, G - 2_000)), frag, lens, "rescue", hard="right" if odd else "left")
                frag = int(rng.integers(900, 1_150))
                add(o, odd, int(rng.integers(0, 30)), frag, (MAX_LEN, 400), "start", hard="left")
                add(o, odd, G - frag - int(rng.integers(0, 30)), frag, (450, MAX_LEN), "end", hard="right")
                add(o, odd, FAMILY[odd] + int(rng.integers(0, 80)), 700, (300, 320), "family")
                continue
            for _ in range(2):
                frag = int(rng.integers(250, 450))
                add(o, odd, int(rng.integers(0, 30)), frag, (100, 100), "start", hard="left")
                frag = int(rng.integers(250, 450))
                add(o, odd, G - frag - int(rng.integers(0, 30)), frag, (100, 100), "end", hard="right")
            for frag in (MINF - 1, MINF, MAXF, MAXF + 1):             # exact mates: their begins are end - length exactly
                add(o, odd, int(rng.integers(1_000, G - 2_000)), frag, (100, 70) if odd else (70, 100), "limit", rate=0.0)
            for _ in range(2):                                          # below min_frag: rescued from each other
                add(o, odd, int(rng.integers(1_000, G - 2_000)), int(rng.integers(130, 190)), (60, 60), "short")
            for lens in ((33, 250), (150, 60)):
                add(o, odd, int(rng.integers(1_000, G - 2_000)), int(rng.integers(300, 480)), lens, "unequal", hard="left" if odd else None)
            # an exact mate longer than max_frag anchoring a substituted one: its --no-overlap window is empty
            add(o, odd, int(rng.integers(1_000, G - 2_000)), int(rng.integers(520, 560)), (505 + 7 * odd, 100) if odd else (100, 505),
                "longmate", hard=1 - odd, rate=0.0)
            for h in ("left", "right"):
                add(o, odd, int(rng.integers(1_000, G - 2_000)), int(rng.integers(250, 450)), (100, 100), "n4", hard=h, n_rate=0.03)
            for c in (0, 1):
                add(o, odd, FAMILY[(2 * odd + c) % 4] + int(rng.integers(0, UNIT - 460)), int(rng.integers(250, 450)), (100, 100), "family")
            for _ in range(2):                                          # mate 2 from a far-away locus: discordant when both are unique
                (a, _b), _lm = mates(g, o, odd, int(rng.integers(1_000, 60_000)), 300, (100, 100))
                q = int(rng.integers(170_000, G - 1_000))
                m1.append(mutate(a, 0.01, rng)); m2.append(mutate(g[q:q + 100] if odd else rc(g[q:q + 100]), 0.01, rng))
                kind.append("elsewhere"); frags.append(0)
            add(o, odd, int(rng.integers(1_000, G - 2_000)), int(rng.integers(250, 450)), (100, 100), "plain")
    return m1 + m2, np.array(kind), np.array(frags)


def make_world(long_mates, seed):
    require_gpu()
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, G).astype(np.uint8)
    unit = rng.integers(0, 4, UNIT).astype(np.uint8)
    for st in FAMILY:
        g[st:st + UNIT] = unit
    reads, kind, frags = plant(g, rng, long_mates)
    O = orc.Oracle()
    idx = O.build_index(g)
    gw = torch.from_numpy(nb.pack_symbols(g, bits=2, big_endian=True, pad_words=8).view(np.int32)).cuda()
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    bits = 2 if long_mates else 4
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)
    K = (int(lens.max()) - SEED_LEN) // SEED_INTERVAL + 1
    return dict(O=O, g=g, gw=gw, idx=idx, fmi=fmi, reads=reads, quals=quals, kind=kind, frags=frags, n=len(kind), lens=lens, rs=rs,
                bits=bits, cap=2 * K * MAX_SEED_HITS * len(reads) + 1024, se={}, se_tb=None)


@pytest.fixture(scope="module")
def world():
    return make_world(False, 2024)


@pytest.fixture(scope="module")
def long_world():
    return make_world(True, 512)


def make_params(w, qual=False, dedup=True):
    kw = dict(seed_len=SEED_LEN, seed_interval=SEED_INTERVAL, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=MAX_SEED_HITS,
              dedup_jobs=dedup)
    if qual:
        return nb.SeedExtendParams(scheme=aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3), read_quals=torch.from_numpy(np.concatenate(w["quals"])).cuda(),
                                   **kw)
    return nb.SeedExtendParams(scheme=aln.SimpleGotohScheme(2, -2, -5, -3), **kw)


_MQ = []


def mq():
    if not _MQ:
        _MQ.append(MapqParams.local(MAX_LEN))
    return _MQ[0]


def run(w, pair, qual=False, dedup=True, mapq=True, traceback=False, path=None):
    if path is not None:
        nb.lib().nvb_debug_pipeline_path(path)
    try:
        ws = nb.seed_extend_paired(w["fmi"], w["gw"], w["rs"], make_params(w, qual, dedup), pair, hit_capacity=w["cap"],
                                   mapq=mq() if mapq else None, traceback=traceback)
        torch.cuda.synchronize()
    finally:
        if path is not None:
            nb.lib().nvb_debug_pipeline_path(0)
    kept, total, _ = (int(v) for v in ws.n_hits.cpu())
    assert kept == total                                              # the oracle assumes no hit is dropped
    keys = PAIR_KEYS + (MAPQ_KEYS if mapq else ()) + (TB_KEYS if traceback else ())
    return {k: getattr(ws, k).cpu().numpy().copy() for k in keys}, ws


def single_end(w, qual):
    """the oracle's single-end composition of every mate, computed once per scheme"""
    if qual not in w["se"]:
        w["se"][qual] = seed_extend_oracle(w["O"], w["idx"], w["g"], w["reads"], make_params(w, qual), quals=w["quals"] if qual else None)
    return w["se"][qual]


def oracle(w, pair, qual=False, mapq=True):
    se = single_end(w, qual)
    q = w["quals"] if qual else None
    with mock.patch.object(pipeline_oracle, "seed_extend_oracle", lambda *a, **k: se):
        if mapq:
            return ppo.pair_mapq_oracle(w["O"], w["idx"], w["g"], w["reads"], make_params(w, qual), pair, w["n"], mq().min_score.cpu().numpy(),
                                        mq().match_bonus, quals=q)
        return ppo.seed_extend_paired_oracle(w["O"], w["idx"], w["g"], w["reads"], make_params(w, qual), pair, w["n"], quals=q)


def compare(got, want, keys, what=()):
    for k in keys:
        g = got[k].astype(np.int64)
        wv = np.asarray(want[k], np.int64).reshape(g.shape)
        if k in ("mate_pos", "second_mate_pos"):                            # device outputs are int32 views of uint32
            g, wv = g & 0xFFFFFFFF, wv & 0xFFFFFFFF
        bad = np.argwhere(g != wv)
        assert len(bad) == 0, (what, k, bad[:5].tolist(), g[tuple(bad[0])], wv[tuple(bad[0])])


def single_best(w, qual=False):
    """(has, score, strand, begin, end) of every mate's single-end best, as the paired stage frames it"""
    se = single_end(w, qual)
    bh = best_hits(se, len(w["reads"]))
    out = []
    for r, h in enumerate(bh):
        if h < 0:
            out.append((False, INT_MIN, 0, 0, 0)); continue
        end = int(se["hit_window"][h][0] + se["hit_sink"][h][0])
        out.append((True, int(se["hit_score"][h]), int(se["hit_string"][h]) % 2, max(end - len(w["reads"][r]), 0), end))
    return out


def coverage(w, pair, want, qual=False):
    """how often each planted edge happened under pair (windows from the single-end bests, as the paired stage computes them)"""
    policy, overlap = pair.policy, pair.overlap
    n, lens = w["n"], w["lens"]
    sb = single_best(w, qual)
    flags = np.asarray(want["pair_flags"])
    c = dict(clip0=0, clipG=0, rescued_clip0=0, rescued_clipG=0, empty=0, at_min=0, at_max=0, rescued_short=0, second=0, n4_rescued=0,
             unequal_paired=0)
    for p in range(n):
        m = [sb[p], sb[n + p]]
        if m[0][0] and m[1][0] and ppo.concordant(policy, overlap, m[0][2:], m[1][2:], pair.min_frag, pair.max_frag):
            continue
        for a in range(2):
            has, s, t, b, e = m[a]
            if not has or s < pair.min_mate_score:
                continue
            wb, we, _ = ppo.rescue_window(policy, overlap, a, t, b, e, pair.max_frag, G)
            left, _ = ppo.frame(policy, a, t)
            rescued_here = flags[p] == (2 if a == 1 else 4)
            if we == wb:
                c["empty"] += 1
            elif left and e < pair.max_frag:
                c["clip0"] += 1; c["rescued_clip0"] += int(rescued_here)
            elif not left and b + pair.max_frag > G:
                c["clipG"] += 1; c["rescued_clipG"] += int(rescued_here)
    pos = np.asarray(want["mate_pos"], np.int64).reshape(2, n)
    for p in range(n):
        if flags[p] not in (1, 2, 4):
            continue
        e = pos[:, p]
        b = np.maximum(e - np.array([lens[p], lens[n + p]], np.int64), 0)
        frag = int(e.max() - b.min())
        if flags[p] == 1:
            c["at_min"] += int(frag == pair.min_frag and pair.min_frag > 0)
            c["at_max"] += int(frag == pair.max_frag)
        else:
            c["rescued_short"] += int(frag < pair.min_frag)
            c["n4_rescued"] += int(w["kind"][p] == "n4")
        c["unequal_paired"] += int(w["kind"][p] == "unequal")
    if "second_pair_score" in want:
        c["second"] = int((np.asarray(want["second_pair_score"]) != INT_MIN).sum())
    return c


def assert_covered(c, pair, what):
    need = ["rescued_clip0", "rescued_clipG", "at_max", "second", "unequal_paired"]
    need += ["at_min", "rescued_short"] if pair.min_frag > 0 else []
    need += ["empty"] if not pair.overlap else []
    need += ["n4_rescued"] if what[0] != "long" else []
    print("coverage", what, c, flush=True)
    assert all(c[k] > 0 for k in need), (what, {k: c[k] for k in need})


# ---- traceback and BAM ------------------------------------------------------------------------------------------------------------------

def se_traceback(w):
    if w["se_tb"] is None:
        se = nb.seed_extend(w["fmi"], w["gw"], w["rs"], make_params(w), hit_capacity=w["cap"], traceback=True)
        torch.cuda.synchronize()
        w["se_tb"] = dict(ops=se.best_ops.cpu().numpy(), n_ops=se.best_n_ops.cpu().numpy(), begin=host_u32(se.best_begin),
                          pos=host_u32(se.best_pos), strand=se.best_strand.cpu().numpy())
    return w["se_tb"]


def check_traceback(w, pair, got, ws):
    """mates that keep their single-end best: its traceback; rescued mates: the full traceback of the policy's window (strand of the
    policy); unaligned mates: none; every aligned mate replays to its score and end.  Returns (rescued mates, clipped windows among them)"""
    n, reads = w["n"], w["reads"]
    se = se_traceback(w)
    flags, mops, mn, mbeg = got["pair_flags"], got["mate_ops"], got["mate_n_ops"], got["mate_begin"].view(np.uint32)
    rescued = []
    for p in range(n):
        for m in range(2):
            r = m * n + p
            if flags[p] in (2, 4) and m == (0 if flags[p] == 2 else 1):
                rescued.append((p, m)); continue
            if np.uint32(got["mate_pos"][m, p]) == NONE:
                assert mn[m, p] == 0 and tuple(mbeg[m, p]) == (NONE, NONE), (p, m); continue
            assert mn[m, p] == se["n_ops"][r] and np.array_equal(mbeg[m, p], se["begin"][r]), (p, m)
            assert np.array_equal(mops[m, p, :mn[m, p]], se["ops"][r, :se["n_ops"][r]]), (p, m)
    pats, t_off, t_len, clipped = [], [], [], 0
    for p, o in rescued:
        a = 1 - o
        ra, ro = a * n + p, o * n + p
        end = int(se["pos"][ra])
        to, te, ot = ppo.rescue_window(pair.policy, pair.overlap, a, int(se["strand"][ra]), max(end - len(reads[ra]), 0), end, pair.max_frag, G)
        assert got["mate_strand"][o, p] == ot, (p, o)
        clipped += int(to == 0 or te == G)
        pats.append(strand_string(reads[ro], w["quals"][ro], ot)[0]); t_off.append(to); t_len.append(te - to)
    if rescued:
        lens = np.array([len(x) for x in pats], np.uint32)
        P = PackedStringSet.from_symbols(np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32), lens, bits=w["bits"])
        T = PackedStringSet.from_symbols(w["g"], np.array(t_off, np.uint32), np.array(t_len, np.uint32), bits=2)
        tb = aln.batch_alignment_traceback(aln.make_gotoh_aligner(aln.LOCAL, make_params(w).scheme), P, T, max_ops=ws.max_ops)
        torch.cuda.synchronize()
        t_ops, t_n, t_src, t_sink = tb["ops"].cpu().numpy(), host_u32(tb["n_ops"]), host_u32(tb["source"]), host_u32(tb["sink"])
        for i, (p, o) in enumerate(rescued):
            assert int(tb["score"][i]) == got["mate_score"][o, p] and t_off[i] + t_sink[i][0] == np.uint32(got["mate_pos"][o, p]), (p, o)
            assert mn[o, p] == t_n[i] and tuple(mbeg[o, p]) == (t_off[i] + t_src[i][0], t_src[i][1]), (p, o)
            assert np.array_equal(mops[o, p, :t_n[i]], t_ops[i, :t_n[i]]), (p, o)
    for p in range(n):
        for m in range(2):
            if np.uint32(got["mate_pos"][m, p]) == NONE:
                continue
            r = m * n + p
            pat, _ = strand_string(reads[r], w["quals"][r], int(got["mate_strand"][m, p]))
            assert replay(mops[m, p], mn[m, p], mbeg[m, p], pat, None, w["g"], make_params(w).scheme) == (int(got["mate_score"][m, p]),
                                                                                                       int(got["mate_pos"][m, p])), (p, m)
    return len(rescued), clipped


def check_bam(w, got, ws):
    """finish -> bam_records -> sam_text of every pair equal bam_oracle and sam_oracle; returns the discordant records with both mates
    placed"""
    n = w["n"]
    f = nb.finish_alignments(w["gw"], w["rs"], ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    cut = FAMILY[1] + 37                                                # a contig boundary inside the repeat family
    contigs = nb.ContigTable(["chrA", "chrB"], [cut, G - cut])
    names = nb.numbered_names(n, "pp")
    recs = nb.bam_records(ws, f, w["rs"], contigs, names)
    torch.cuda.synchronize()
    off = recs.offsets.cpu().numpy()
    raw = recs.data[:int(off[-1])].cpu().numpy().tobytes()
    inp = dict(reads=w["reads"], quals=None, n_ops=got["mate_n_ops"].reshape(-1).astype(np.uint32),
               begin=got["mate_begin"].reshape(-1, 2).view(np.uint32), strand=got["mate_strand"].reshape(-1).astype(np.uint8),
               cigar=host_u32(f.cigar), n_cigar=host_u32(f.n_cigar), md=f.md.cpu().numpy(), md_len=host_u32(f.md_len), edits=host_u32(f.edits),
               score=got["mate_score"].reshape(-1).astype(np.int32), mapq=got["mate_mapq"].reshape(-1).astype(np.uint8),
               second=got["mate_second_score"].reshape(-1).astype(np.int32), pair_flags=got["pair_flags"].astype(np.uint32),
               contig_begin=contigs.begin, contig_names=contigs.names, contig_lengths=list(contigs.lengths), names=names)
    want, cnt = bam_oracle.records(inp)
    assert len(want) == 2 * n and len(off) == 2 * n + 1
    disc = 0
    for k, (wb, sam) in enumerate(want):
        assert raw[off[k]:off[k + 1]] == wb, (k, sam)
        flag = int(sam.split("\t")[1])
        if got["pair_flags"][k // 2] == nb.PAIR_DISCORDANT and not flag & 0xC:
            assert flag & 0x1 and not flag & 0x2
            disc += 1
    t = nb.sam_text(recs, contigs)
    torch.cuda.synchronize()
    lines, bad = sam_oracle.text(raw, off, contigs.names)
    so = t.offsets.cpu().numpy()
    text = t.data[:int(so[-1])].cpu().numpy().tobytes()
    assert t.rejected.cpu().numpy().view(np.uint32).tolist() == bad == [0, NONE]
    assert [text[so[i]:so[i + 1]] for i in range(2 * n)] == lines
    return disc


# ---- the tests ---------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("overlap", [True, False])
@pytest.mark.parametrize("min_frag", [0, MINF])
def test_edges_vs_oracle(world, policy, overlap, min_frag):
    w = world
    what = ("edges", policy, overlap, min_frag)
    pair = nb.PairParams(min_frag=min_frag, max_frag=MAXF, min_mate_score=60, policy=policy, overlap=overlap)
    want = oracle(w, pair)
    got, _ = run(w, pair)
    compare(got, want, PAIR_KEYS + MAPQ_KEYS, what)
    compare(run(w, pair, mapq=False)[0], want, PAIR_KEYS, what + ("no mapq",))
    compare(run(w, pair, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("per hit",))
    compare(run(w, pair, dedup=False)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("no dedup",))
    compare(run(w, pair, dedup=False, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("per hit, no dedup",))
    assert_covered(coverage(w, pair, want), pair, what)
    # a rescue capacity that cuts the job list: the first jobs in pair order run, the rest are reported wanted
    # (the largest of wanted / 2, / 4, / 8 and 4 that drops a rescue)
    ran, wanted = (int(v) for v in want["n_rescue"])
    assert ran == wanted and wanted >= 8
    for cap in (wanted // 2, wanted // 4, wanted // 8, 4):
        capped = nb.PairParams(min_frag=min_frag, max_frag=MAXF, min_mate_score=60, policy=policy, overlap=overlap, rescue_capacity=cap)
        want_c = oracle(w, capped)
        if (np.asarray(want_c["pair_flags"]) != np.asarray(want["pair_flags"])).any():
            break
    assert tuple(want_c["n_rescue"]) == (cap, wanted) and (np.asarray(want_c["pair_flags"]) != np.asarray(want["pair_flags"])).any()
    compare(run(w, capped)[0], want_c, PAIR_KEYS + MAPQ_KEYS, what + ("capped",))


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("mixed", [True, False])
def test_discordant_traceback_bam(world, policy, mixed):
    """discordant pairs, with and without --no-mixed, traced; their finish, BAM records and SAM lines"""
    w = world
    what = ("discordant", policy, mixed)
    overlap = policy in ("fr", "rr")
    pair = nb.PairParams(min_frag=MINF, max_frag=MAXF, min_mate_score=60, policy=policy, overlap=overlap, discordant=True, mixed=mixed)
    want = oracle(w, pair)
    got, ws = run(w, pair, traceback=True)
    compare(got, want, PAIR_KEYS + MAPQ_KEYS, what)
    compare(run(w, pair, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("per hit",))
    flags = got["pair_flags"]
    disc = flags == nb.PAIR_DISCORDANT
    assert disc[w["kind"] == "elsewhere"].sum() >= 3 and not disc[w["kind"] == "family"].any(), what
    if not mixed:
        assert (flags == nb.PAIR_UNPAIRED).sum() > 0
    n_resc, clipped = check_traceback(w, pair, got, ws)
    n_disc = check_bam(w, got, ws)
    c = coverage(w, pair, want)
    c.update(rescued_traces=n_resc, clipped_traces=clipped, discordant_records=n_disc)
    assert_covered(c, pair, what)
    assert n_resc >= 10 and clipped > 0 and n_disc > 0, c


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_quality_scheme(world, policy):
    w = world
    what = ("quality", policy)
    pair = nb.PairParams(min_frag=MINF, max_frag=MAXF, min_mate_score=50, policy=policy, overlap=policy in ("rf", "ff"))
    want = oracle(w, pair, qual=True)
    compare(run(w, pair, qual=True)[0], want, PAIR_KEYS + MAPQ_KEYS, what)
    compare(run(w, pair, qual=True, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("per hit",))
    assert_covered(coverage(w, pair, want, qual=True), pair, what)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", ("rf", "ff"))
def test_long_mates(long_world, policy):
    """300-512 bp mates (the traceback's limit), rescue windows clipped at both ends, under RF and FF with and without overlap"""
    w = long_world
    for overlap in (True, False):
        what = ("long", policy, overlap)
        pair = nb.PairParams(min_frag=MINF, max_frag=1_200, min_mate_score=60, policy=policy, overlap=overlap, discordant=True)
        want = oracle(w, pair)
        got, ws = run(w, pair, traceback=True)
        compare(got, want, PAIR_KEYS + MAPQ_KEYS, what)
        compare(run(w, pair, path=1)[0], want, PAIR_KEYS + MAPQ_KEYS, what + ("per hit",))
        n_resc, clipped = check_traceback(w, pair, got, ws)
        c = coverage(w, pair, want)
        c.update(rescued_traces=n_resc, clipped_traces=clipped, discordant_records=check_bam(w, got, ws))
        need = ["rescued_clip0", "rescued_clipG", "second"]
        print("coverage", what, c, flush=True)
        assert all(c[k] > 0 for k in need) and n_resc >= 5 and clipped > 0, (what, c)
