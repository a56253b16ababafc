"""Oracle composition of paired-end seed + extend under every pairing policy and option (test infrastructure): nvb_pair_params.policy
(FR, RF, FF, RR) and flags (no overlap, discordant pairs, no mixed) as include/nvbio_b200.h states them.  The pinned FR oracles
(tests/pipeline_oracle.py, tests/pair_mapq_oracle.py, tests/paired_reseed_oracle.py) stay as they are; this module restates the
paired stage with the policy and reuses their single-end composition, MAPQ and helpers.  With a PairParams at its defaults every
function here gives the answers of the FR oracle it generalises.

  - frame / concordant / rescue_window: nvBowtie's frame_opposite_mate, the concordance test and the opposite-mate window;
  - seed_extend_paired_oracle: nvb_seed_extend_paired;
  - second_pair / rescue_jobs / pair_mapq_oracle: nvb_seed_extend_paired_mapq (second-best pair by brute force);
  - seed_extend_paired_reseed_oracle: nvb_seed_extend_paired_reseed, tests/paired_reseed_oracle.py's composition with the two paired
    oracles above in place of the FR ones.

The single-end stage is looked up as pipeline_oracle.seed_extend_oracle at call time, so that a caller may substitute it (the reseed
composition answers it with the union of its rounds)."""
from unittest import mock
import numpy as np
from tests import pipeline_oracle, pair_mapq_oracle as pmo, paired_reseed_oracle
from tests.mapq_oracle import bowtie_mapq2, mapq_oracle, INT_MIN
from tests.pipeline_oracle import _scheme_args, best_hits, EMPTY_SINK
from tests.pair_mapq_oracle import _distinct, NONE_TIE


def pair_options(pair):
    """(policy, overlap, discordant, mixed) of a PairParams; objects without these fields are the FR pairing of before"""
    return (getattr(pair, "policy", "fr"), getattr(pair, "overlap", True), getattr(pair, "discordant", False), getattr(pair, "mixed", True))


def frame(policy, a, t):
    """(left, strand) of the other mate of anchor mate a (0 = mate 1) aligned on strand t: nvBowtie's frame_opposite_mate restated
    (alignment_utils.h:61-98, anchor_fw = t == 0)"""
    fw, a1 = t == 0, a == 0
    left, ofw = {"ff": (a1 != fw, fw), "rr": (a1 == fw, fw), "rf": (fw, not fw), "fr": (not fw, not fw)}[policy]
    return bool(left), 0 if ofw else 1


def concordant(policy, overlap, m1, m2, min_frag, max_frag):
    """m1 / m2 = (strand, begin, end) of mate 1 / mate 2: the concordance test of include/nvbio_b200.h (nvb_pair_params)"""
    left, o = frame(policy, 0, m1[0])
    if m2[0] != o:
        return False
    (_, lb, le), (_, rb, re_) = (m2, m1) if left else (m1, m2)
    return lb <= rb and le <= re_ and re_ > lb and min_frag <= re_ - lb <= max_frag and (overlap or le <= rb)


def rescue_window(policy, overlap, a, t, b, e, max_frag, glen):
    """(window begin, window end, strand of the other mate) of the opposite-mate job of anchor mate a on strand t at [b, e)"""
    left, o = frame(policy, a, t)
    if left:
        wb, we = max(e - max_frag, 0), (e if overlap else b)
    else:
        wb, we = (b if overlap else e), min(b + max_frag, glen)
    return wb, max(we, wb), o


def seed_extend_paired_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, quals=None, unique=None):
    """Oracle composition of nvb_seed_extend_paired under pair's policy and options: pipeline_oracle's single-end composition for the
    2*n_pairs mates, the pairing rules of include/nvbio_b200.h restated in Python, and the opposite-mate rescue scored by the oracle's
    full-matrix Gotoh.  reads: mate 1 of every pair, then mate 2.  unique[r]: read r's best alignment reaches its min score and has no
    single-end second (the MAPQ stage's; required with pair.discordant).  Returns dict(pair_score, pair_flags, mate_score[2,n],
    mate_pos[2,n], mate_strand[2,n], n_rescue)."""
    policy, overlap, discordant, mixed = pair_options(pair)
    if discordant and unique is None:
        raise ValueError("discordant pairs need the single-end second best of the MAPQ stage (pair_mapq_oracle)")
    se = pipeline_oracle.seed_extend_oracle(O, idx, genome_sym, reads, params, quals=quals)
    glen = idx.n
    strands = 2
    best_h = best_hits(se, len(reads), strands)
    INT_MIN = -2**31

    def mate(r):
        h = best_h[r]
        if h < 0:
            return dict(has=False, score=INT_MIN, strand=0, beg=0xFFFFFFFF, end=0xFFFFFFFF, len=0)
        s = int(se["hit_string"][h])
        ln = len(reads[r])
        end = int(se["hit_window"][h][0] + se["hit_sink"][h][0])
        return dict(has=True, score=int(se["hit_score"][h]), strand=s % strands, beg=max(end - ln, 0), end=end, len=ln)

    cap = 2 * n_pairs if pair.rescue_capacity is None else pair.rescue_capacity
    pair_score = np.full(n_pairs, INT_MIN, np.int64); pair_flags = np.zeros(n_pairs, np.int64)
    mate_score = np.full((2, n_pairs), INT_MIN, np.int64); mate_pos = np.full((2, n_pairs), 0xFFFFFFFF, np.int64)
    mate_strand = np.zeros((2, n_pairs), np.int64)
    jobs = []          # (pair, anchor, pattern symbols, window begin, window length)
    for p in range(n_pairs):
        m = [mate(p), mate(n_pairs + p)]
        for k in range(2):
            mate_score[k, p], mate_pos[k, p], mate_strand[k, p] = m[k]["score"], m[k]["end"], m[k]["strand"]
        conc = m[0]["has"] and m[1]["has"] and concordant(policy, overlap, (m[0]["strand"], m[0]["beg"], m[0]["end"]),
                                                          (m[1]["strand"], m[1]["beg"], m[1]["end"]), pair.min_frag, pair.max_frag)
        if conc:
            pair_score[p] = m[0]["score"] + m[1]["score"]; pair_flags[p] = 1
            continue
        for a in range(2):
            if not (m[a]["has"] and m[a]["score"] >= pair.min_mate_score):
                continue
            o = reads[(1 - a) * n_pairs + p]
            oq = quals[(1 - a) * n_pairs + p] if quals is not None else None
            to, te, ot = rescue_window(policy, overlap, a, m[a]["strand"], m[a]["beg"], m[a]["end"], pair.max_frag, glen)
            if ot == 1:
                pat = np.where(o < 4, 3 - o, o)[::-1].astype(np.uint8)
                pq = oq[::-1] if oq is not None else None
            else:
                pat = o
                pq = oq
            if te - to >= 1 and len(pat) >= 1:
                jobs.append((p, a, pat, to, te - to, pq))
    wanted = len(jobs)
    run = jobs[:cap]
    if run:
        pats = np.concatenate([j[2] for j in run])
        p_len = np.array([len(j[2]) for j in run], np.uint32)
        p_off = (np.cumsum(p_len) - p_len).astype(np.uint32)
        t_off = np.array([j[3] for j in run], np.uint32); t_len = np.array([j[4] for j in run], np.uint32)
        scheme, qtab = _scheme_args(params.scheme)
        rs, rx, _ = O.gotoh_full(params.type, scheme, pats, p_off, p_len, genome_sym, t_off, t_len,
                                 qual=np.concatenate([j[5] for j in run]) if quals is not None else None, qtab=qtab)
        cand = {}
        for (p, a, _, to, _, _), s, x in zip(run, rs, rx):
            if int(s) < pair.min_mate_score:
                continue
            tot = int(mate_score[a, p]) + int(s)
            if p not in cand or tot > cand[p][0]:
                cand[p] = (tot, a, int(s), to + int(x))
        for p, (tot, a, s, pos) in cand.items():
            o = 1 - a
            pair_score[p] = tot; pair_flags[p] = 2 if o == 0 else 4
            mate_score[o, p] = s; mate_pos[o, p] = pos; mate_strand[o, p] = frame(policy, a, int(mate_strand[a, p]))[1]
    for p in np.flatnonzero(pair_flags == 0):
        if discordant and unique[p] and unique[n_pairs + p]:
            pair_score[p] = mate_score[0, p] + mate_score[1, p]; pair_flags[p] = 8
        elif not mixed:
            mate_score[:, p], mate_pos[:, p], mate_strand[:, p] = INT_MIN, 0xFFFFFFFF, 0
    return dict(pair_score=pair_score, pair_flags=pair_flags, mate_score=mate_score, mate_pos=mate_pos, mate_strand=mate_strand,
                n_rescue=(len(run), wanted))


def second_pair(c1, c2, len1, len2, star, min_frag, max_frag, rescues=(), policy="fr", overlap=True):
    """c1 / c2: mate 1's / mate 2's candidates (score, strand, end, tie), already at or above the min score; star = ((end, strand) of P*'s
    mate 1, of its mate 2); rescues: (anchor mate, pair score, anchor end, anchor strand, anchor tie, rescued end[, rescued strand], the
    anchor's opposite strand when not given).  Every combination of one candidate of each mate is tested for concordance under policy /
    overlap (no merging, no search).  Returns (score, ((end1, strand1), (end2, strand2))) of the second-best pair, or None."""
    A = np.array(c1, np.int64).reshape(-1, 4)[:, None, :]
    B = np.array(c2, np.int64).reshape(-1, 4)[None, :, :]
    e1, t1, e2, t2 = A[..., 2], A[..., 1], B[..., 2], B[..., 1]
    b1, b2 = np.where(e1 > len1, e1 - len1, 0), np.where(e2 > len2, e2 - len2, 0)
    fr = [frame(policy, 0, t) for t in (0, 1)]                     # mate 1's framing on either strand
    left1, o1 = np.array([f[0] for f in fr])[t1], np.array([f[1] for f in fr])[t1]
    lb, le, rb, re_ = np.where(left1, b2, b1), np.where(left1, e2, e1), np.where(left1, b1, b2), np.where(left1, e1, e2)
    ok = (t2 == o1) & (lb <= rb) & (le <= re_) & (re_ > lb) & (re_ - lb >= min_frag) & (re_ - lb <= max_frag) & (overlap | (le <= rb))
    ok = np.broadcast_to(ok, (A.shape[0], B.shape[1]))
    i, j = np.nonzero(ok)
    S = (A[i, 0, 0] + B[0, j, 0]).tolist()
    cols = [S, A[i, 0, 3].tolist(), B[0, j, 3].tolist(), A[i, 0, 2].tolist(), A[i, 0, 1].tolist(), B[0, j, 2].tolist(), B[0, j, 1].tolist()]
    for r in rescues:
        a, sc, ae, at, ai, oe = r[:6]
        ot = r[6] if len(r) > 6 else 1 - at
        m1, m2 = ((ae, at, ai), (oe, ot, NONE_TIE)) if a == 0 else ((oe, ot, NONE_TIE), (ae, at, ai))
        for c, v in zip(cols, (sc, m1[2], m2[2], m1[0], m1[1], m2[0], m2[1])):
            c.append(v)
    S, I1, I2, E1, T1, E2, T2 = (np.array(c, np.int64) for c in cols)
    keep = _distinct(E1, T1, star[0][0], star[0][1], len1) | _distinct(E2, T2, star[1][0], star[1][1], len2)
    if not keep.any():
        return None
    k = np.flatnonzero(keep)[np.lexsort((I2[keep], I1[keep], -S[keep]))[0]]
    return int(S[k]), ((int(E1[k]), int(T1[k])), (int(E2[k]), int(T2[k])))


def rescue_jobs(O, idx, genome_sym, reads, params, pair, n_pairs, single, redo, quals=None):
    """every opposite-mate job of the paired stage as the header states it, scored by the oracle's full-matrix Gotoh: (pair, anchor,
    window begin, score, sink.x, rescued strand) of the first rescue_capacity jobs, and the number wanted.  single: the mates'
    single-end bests (mapq_oracle); redo[p]: the pair was not concordant as it stood"""
    policy, overlap, _, _ = pair_options(pair)
    jobs = []
    for p in np.flatnonzero(redo):
        for a in range(2):
            ra = a * n_pairs + p
            if single["best_score"][ra] == INT_MIN or single["best_score"][ra] < pair.min_mate_score:
                continue
            end, ln = int(single["best_pos"][ra]), len(reads[ra])
            o = reads[(1 - a) * n_pairs + p]
            oq = quals[(1 - a) * n_pairs + p] if quals is not None else None
            to, te, ot = rescue_window(policy, overlap, a, int(single["best_strand"][ra]), max(end - ln, 0), end, pair.max_frag, idx.n)
            if ot == 1:
                pat, pq = np.where(o < 4, 3 - o, o)[::-1].astype(np.uint8), (oq[::-1] if oq is not None else None)
            else:
                pat, pq = o, oq
            if te - to >= 1 and len(pat) >= 1:
                jobs.append((int(p), a, pat, to, te - to, pq, ot))
    cap = 2 * n_pairs if pair.rescue_capacity is None else pair.rescue_capacity
    run = jobs[:cap]
    if not run:
        return [], len(jobs)
    p_len = np.array([len(j[2]) for j in run], np.uint32)
    scheme, qtab = _scheme_args(params.scheme)
    rs, rx, _ = O.gotoh_full(params.type, scheme, np.concatenate([j[2] for j in run]), (np.cumsum(p_len) - p_len).astype(np.uint32), p_len,
                             genome_sym, np.array([j[3] for j in run], np.uint32), np.array([j[4] for j in run], np.uint32),
                             qual=np.concatenate([j[5] for j in run]) if quals is not None else None, qtab=qtab)
    return [(p, a, to, int(s), int(x), ot) for (p, a, _, to, _, _, ot), s, x in zip(run, rs, rx)], len(jobs)


def pair_mapq_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, min_score, match_bonus, quals=None):
    """the oracle composition of every nvb_seed_extend_paired_mapq output (int64 arrays; mates as [2, n_pairs]) under pair's policy and
    options"""
    policy, overlap, _, mixed = pair_options(pair)
    se = pipeline_oracle.seed_extend_oracle(O, idx, genome_sym, reads, params, quals=quals)
    lens = np.array([len(r) for r in reads], np.int64)
    ms = np.asarray(min_score, np.int64)
    single = mapq_oracle(se, lens, 2, ms, match_bonus)
    # a discordant pair's mates: aligned at or above the min score, no single-end second
    unique = (single["best_score"] != INT_MIN) & (single["best_score"] >= ms[lens]) & (single["second_score"] == INT_MIN)
    pe = seed_extend_paired_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, quals=quals, unique=unique)
    best_h = best_hits(se, len(reads))                             # every read's best hit (its tie index): max score, then smallest hit
    rescues, wanted = rescue_jobs(O, idx, genome_sym, reads, params, pair, n_pairs, single, pe["pair_flags"] != 1, quals=quals)
    assert (len(rescues), wanted) == tuple(pe["n_rescue"])         # the same jobs as the paired composition ran
    end = se["hit_window"][:, 0] + se["hit_sink"][:, 0] if len(se["hit_string"]) else np.zeros(0, np.int64)
    cands = [[] for _ in reads]
    for h, s in enumerate(se["hit_string"]):
        r = int(s) // 2
        if se["hit_sink"][h][0] != EMPTY_SINK and se["hit_score"][h] >= ms[lens[r]]:
            cands[r].append((int(se["hit_score"][h]), int(s) % 2, int(end[h]), h))
    resc = {}
    for p, a, to, rs, x, ot in rescues:
        if rs >= pair.min_mate_score and rs >= ms[lens[(1 - a) * n_pairs + p]]:
            ra = a * n_pairs + p
            resc.setdefault(p, []).append((a, int(se["hit_score"][best_h[ra]]) + rs, int(single["best_pos"][ra]), int(single["best_strand"][ra]),
                                           int(best_h[ra]), to + x, ot))
    out = dict(pair_score=pe["pair_score"], pair_flags=pe["pair_flags"], mate_score=pe["mate_score"], mate_pos=pe["mate_pos"],
               mate_strand=pe["mate_strand"], n_rescue=pe["n_rescue"],
               second_pair_score=np.full(n_pairs, INT_MIN, np.int64), second_mate_pos=np.full((2, n_pairs), 0xFFFFFFFF, np.int64),
               second_mate_strand=np.zeros((2, n_pairs), np.int64), mate_second_score=single["second_score"].reshape(2, n_pairs).copy(),
               mate_mapq=single["mapq"].reshape(2, n_pairs).copy())
    for p in range(n_pairs):
        if pe["pair_flags"][p] == 0:
            if not mixed:                                          # both mates reported unaligned
                out["mate_mapq"][:, p] = 0; out["mate_second_score"][:, p] = INT_MIN
            continue
        l1, l2 = int(lens[p]), int(lens[n_pairs + p])
        star = ((int(pe["mate_pos"][0, p]), int(pe["mate_strand"][0, p])), (int(pe["mate_pos"][1, p]), int(pe["mate_strand"][1, p])))
        sp = None if pe["pair_flags"][p] == 8 else second_pair(cands[p], cands[n_pairs + p], l1, l2, star, pair.min_frag, pair.max_frag,
                                                               resc.get(p, ()), policy, overlap)
        if sp is not None:
            out["second_pair_score"][p] = sp[0]
            for k in range(2):
                out["second_mate_pos"][k, p], out["second_mate_strand"][k, p] = sp[1][k]
        q = bowtie_mapq2(pe["pair_score"][p], sp is not None, sp[0] if sp is not None else 0, l1 + l2, match_bonus, ms[l1] + ms[l2])
        out["mate_mapq"][:, p] = int(q)
    return out


def seed_extend_paired_reseed_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, max_reseed, rep_seeds, hit_capacity,
                                     min_score=None, match_bonus=None, quals=None):
    """tests/paired_reseed_oracle.py's composition of nvb_seed_extend_paired_reseed with the pairing under pair's policy: its rounds as
    they are, then seed_extend_paired_oracle / pair_mapq_oracle above on the union of the rounds' hits"""
    with mock.patch.object(pipeline_oracle, "seed_extend_paired_oracle", seed_extend_paired_oracle), \
            mock.patch.object(pmo, "pair_mapq_oracle", pair_mapq_oracle):
        return paired_reseed_oracle.seed_extend_paired_reseed_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, max_reseed, rep_seeds,
                                                                     hit_capacity, min_score=min_score, match_bonus=match_bonus, quals=quals)
